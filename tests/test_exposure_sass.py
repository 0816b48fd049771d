"""The exposure kernels' atomics in the compiled library, read from its SASS with cuobjdump (no device needed): every
one is a reduction nobody waits for (RED in global memory, never an ATOMG whose result is thrown away), and the t = 0
values of the walk are warp-reduced with redux.sync before their one RED per warp."""
import re

from test_sass_guard import kernels  # noqa: F401  (the parsed SASS, a module-scoped fixture)


def _expo(kernels):  # noqa: F811
    out = {k: "\n".join(ls) for k, ls in kernels.items() if "k_expo_" in k}
    assert len(out) == 7, sorted(out)          # op_round, walk<0|1|2>, series, dom_init, dom_max
    return out


def test_no_atomic_with_a_return_value(kernels):  # noqa: F811
    for k, body in _expo(kernels).items():
        assert not re.search(r"ATOMG", body), k


def test_walk_and_max_use_reductions(kernels):  # noqa: F811
    bodies = _expo(kernels)
    walk0 = [b for k, b in bodies.items() if "k_expo_walkILi0E" in k]
    assert walk0 and "REDG" in walk0[0] and "REDUX" in walk0[0]
    assert any("REDG" in b for k, b in bodies.items() if "k_expo_dom_max" in k)
