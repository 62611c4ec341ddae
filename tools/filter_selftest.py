#!/usr/bin/env python3
"""Run gf_cuda_selftest_filter (the certificate of the filtered rolling-shutter pre-pass, on the real MUFU units) for several seeds and
print what it measured.  Needs a GPU."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gyroflow_b200 as g
lib = g.load_library()
tot = [0, 0, 0, 0]
for seed, n_cfg, step in ((2024, 400, 3), (7, 400, 2), (99, 200, 1)):
    out = (C.c_ulonglong * 4)()
    rc = lib.gf_cuda_selftest_filter(0, seed, n_cfg, step, out)
    n, viol, unc, worst = [int(v) for v in out]
    print("seed %d, %d random lenses/matrices/frame sizes, every %d-th pixel: %d pixels in regime, %d violations of the bound, "
          "%.3f %% uncertain, worst |diff| / bound = %.4f (rc %d)" % (seed, n_cfg, step, n, viol, 100.0 * unc / max(n, 1), worst / 1e6, rc))
    tot[0] += n; tot[1] += viol; tot[2] += unc; tot[3] = max(tot[3], worst)
print("total: %d pixels, %d violations, %.3f %% uncertain, worst ratio %.4f; bound = 96u |tv - c| + 4u |c| (rho = 92u = kFilterRho, u = 2^-24)" % (tot[0], tot[1], 100.0 * tot[2] / tot[0], tot[3] / 1e6))
