#!/usr/bin/env python3
"""Wall time of the automatic sync-point choice (gf_cuda_optimal_sync_points) on seeded synthetic 10-minute gyro logs at 2 kHz and 8 kHz.

Each log is timed after one warm-up call, --reps times, by the host clock around the synchronous call (which ends in a stream
synchronise); the median is reported with the card's name and power limit from the same run.  For comparison, a CPU stand-in on all
host threads computes the same band energies with scipy's f32 FFT (workers = all CPUs) and the same band logic, followed by the library's
selection.  It is not the reference (rustfft, one FFT at a time, all spectra kept) and is labelled so.  Prints one JSON line (and writes
it to --out if given).
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.fft

import gyroflow_b200 as g
from tests import np_optsync as npo


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:          # the number still stands; say why the card line is missing
        return "unknown (%s)" % e


def synthetic_log(rate, seconds, seed):
    rng = np.random.default_rng(seed)
    n = int(seconds * rate) + 1
    ts = np.arange(n) * (1000.0 / rate)
    t = ts / 1000.0
    gy = rng.normal(0.0, 2.0, (n, 3))
    for k in range(6):                                   # motion bursts of a few seconds
        t0 = rng.uniform(0, seconds - 10); m = (t >= t0) & (t < t0 + rng.uniform(2, 8))
        gy[m, k % 3] += rng.uniform(50, 300) * np.sin(2 * np.pi * rng.uniform(2, 20) * t[m])
    return ts, gy


def cpu_stand_in(ts, gy, target, workers):
    """scipy f32 FFTs with the reference's band logic, then the library's selection (host)."""
    sr, g64 = npo.resample(ts, gy)
    N = int(npo.round_half_away(sr))
    g32 = g64.astype(np.float32)
    nw = (g32.shape[0] - N) // 16 + 1
    win = npo.blackman(N)
    b = [0, npo.map_to_bin(N, sr, 2.0), npo.map_to_bin(N, sr, 30.0), npo.map_to_bin(N, sr, 2000.0)]
    scale = np.float32(npo.scale_f32(N))
    h = N // 2; k = np.arange(h)
    bands = np.zeros((nw, 3), np.float32)
    chunk = max(1, (64 << 20) // (N * 8 * 3))
    for w0 in range(0, nw, chunk):
        idx = np.arange(w0, min(nw, w0 + chunk)) * 16
        seg = np.lib.stride_tricks.sliding_window_view(g32, N, axis=0)[idx]          # w x 3 x N
        X = scipy.fft.fft(seg * win, axis=-1, workers=workers)
        mag = np.abs(X[..., k] + X[..., N - 1 - k]) * scale
        merged = (mag[:, 0] + mag[:, 1]) + mag[:, 2]
        for i in range(3):
            bands[w0:w0 + len(idx), i] = merged[:, b[i]:b[i + 1]].sum(axis=1)
    return g.optimal_sync_select(bands, sr, N, target)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rates", default="2000,8000")
    ap.add_argument("--seconds", type=float, default=600.0)
    ap.add_argument("--target", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    workers = os.cpu_count() or 1
    result = dict(card=card(), seconds=a.seconds, target=a.target, reps=a.reps, logs=[])
    for i, rate in enumerate(int(r) for r in a.rates.split(",")):
        ts, gy = synthetic_log(rate, a.seconds, 1000 + i)
        sr, N, nr, nw = g.optimal_sync_sizes(ts)
        pts = g.optimal_sync_points(ts, gy, target=a.target)[0]          # warm-up
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            p = g.optimal_sync_points(ts, gy, target=a.target)[0]
            times.append((time.perf_counter() - t0) * 1000.0)
            assert np.array_equal(p, pts)
        row = dict(rate_hz=rate, fft_size=N, samples=int(ts.size), windows=nw, gpu_ms_median=float(np.median(times)),
                   gpu_ms_all=[round(t, 2) for t in times], points_ms=[round(float(x), 3) for x in pts])
        if not a.no_cpu:
            t0 = time.perf_counter()
            cp = cpu_stand_in(ts, gy, a.target, workers)[0]
            row["cpu_stand_in_ms"] = (time.perf_counter() - t0) * 1000.0
            row["cpu_stand_in"] = "scipy f32 FFT on %d threads + the library's selection; not the reference" % workers
            row["cpu_stand_in_points_ms"] = [round(float(x), 3) for x in cp]
        result["logs"].append(row)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
