"""Runs tools/spec_model.c (design model of the speculative assign pass, TEST INFRASTRUCTURE) on a
synthetic configuration and prints the path statistics; asserts the model's decisions equal the oracle's."""
import ctypes, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("BLANCE_NO_NATIVE", "1")
from blance_b200 import synth, tables

def build():
    so = os.path.join(ROOT, "tools", "_spec_model.so")
    src = os.path.join(ROOT, "tools", "spec_model.c")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(os.path.join(ROOT, "oracle", "fast.c"))):
        subprocess.run(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include"), src, "-o", so, "-lm"], check=True)
    return ctypes.CDLL(so)

NAMES = ["steps", "elig", "fast", "slow_sticky", "movers", "inelig", "stale", "t_ge_b0", "list_ok", "list_fail", "list_rebuild", "list_ok_sticky", "asserts_failed",
         "list_fail_k", "xres_ok", "xmax"]
XHIST = ["0", "1", "2", "3-4", "5-8", "9-16", "17-32", "33-64", "65-128", ">128"]

def run(t, H=256, resweeps=2, L=32, Lmin=6):
    lib = build()
    r = tables.PlanResult(t)
    s = t.struct()
    st = (ctypes.c_longlong * 32)()
    t0 = time.time()
    rc = lib.spec_model_plan(ctypes.byref(s), ctypes.byref(r.out), H, resweeps, L, Lmin, st)
    assert rc == 0
    v = list(st)
    d = dict(zip(NAMES, v))
    d["xhist"] = dict(zip(XHIST, v[len(NAMES):len(NAMES) + len(XHIST)]))
    d["seconds"] = time.time() - t0
    return r, d

if __name__ == "__main__":
    P = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    t = synth.make_rebalance(4, P=P)
    t.max_iters = iters
    # "kernel": the speculative kernel's list (up to 63 entries, rebuilt below 4)
    runs = [dict(L=63, Lmin=4)] if "--kernel-list" in sys.argv else [dict(), dict(H=64, resweeps=8), dict(H=1024, resweeps=1), dict(L=16, Lmin=4)]
    for kw in runs:
        r, d = run(t, **kw)
        print(kw, d, flush=True)
