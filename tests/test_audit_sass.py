"""The audit kernels' atomics in the compiled library - read from its SASS with cuobjdump, no device needed: every
one is a reduction nobody waits for (RED / REDG in global memory, never an ATOMG whose result is thrown away), the
scalars and the emptiness test go through redux.sync, and the per-CTA tables are reduced in shared memory."""
import re

import pytest

from test_sass_guard import kernels  # noqa: F401  (the parsed SASS, a module-scoped fixture)


def _audit(kernels):  # noqa: F811
    out = {k: "\n".join(ls) for k, ls in kernels.items() if "k_map_audit" in k or "k_audit_n2n_max" in k}
    assert len(out) == 4, sorted(out)                      # k_map_audit<false|true>, k_map_audit_rules, k_audit_n2n_max
    return out


def test_no_atomic_with_a_return_value(kernels):  # noqa: F811
    for k, body in _audit(kernels).items():
        assert not re.search(r"ATOMG", body), k


@pytest.mark.parametrize("name,ops", [("k_map_audit", ("REDG", "REDUX", "ATOMS")), ("k_map_audit_rules", ("REDG", "REDUX", "ATOMS")),
                                      ("k_audit_n2n_max", ("REDG", "REDUX"))])
def test_instructions(kernels, name, ops):  # noqa: F811
    bodies = [b for k, b in _audit(kernels).items() if re.search(name + r"(I|E)", k)]
    assert bodies
    for body in bodies:
        for op in ops:
            assert op in body, (name, op)
