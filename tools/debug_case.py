import sys, ctypes as C
import os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import gyroflow_b200 as g
from tests import cases, oracle_lib
from tests.test_parity_gpu import run_both
lib = g.load_library()
out = (C.c_ulonglong * 4)()
print("selftest rc", lib.gf_cuda_selftest(0, 1 << 26, 999, out), list(out))
for case in (dict(w=640, h=360, identity=True, rs=False), dict(w=640, h=360)):
    want, got, pix = run_both(case)
    bad = np.argwhere((want != got).reshape(want.shape[0], -1))
    ys, xs = bad[:, 0], bad[:, 1] // 4
    print(case, "mismatch bytes", len(bad), sorted(set(zip(ys.tolist(), xs.tolist())))[:20])
    for (y, x) in sorted(set(zip(ys.tolist(), xs.tolist())))[:6]:
        print(y, x, want[y, 4*x:4*x+4], got[y, 4*x:4*x+4])
