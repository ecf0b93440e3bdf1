#!/usr/bin/env python
"""K5W: long-read consensus against SV reference windows wider than 16377 columns (dgpu_long_needle_ex, the wide-window engine lnw_kernel).

Workload: 512 jobs, consensus of 2-5 kb against windows of 16.4-40 kb (DEL-, DUP- and INV-shaped, 2 % substitutions, 10 % unrelated).

  value       alignments/s from the library's CUDA events around the alignment kernels (median of the timed repetitions)
  tcups       DP cells of both passes ((|cons|+1) x (|ref|+1) each) per second of kernel time, 1e12
  e2e_value   alignments/s of the host-pointer call (copies in and out included)
  cpu_baseline  the reference's longNeedle (oracle/_ref, compiled verbatim) on host cores on the first jobs of the batch, with the thread
                count bounded by host memory (the reference allocates 16 B per DP cell); the GPU alignments of those jobs must equal it

Usage: python tools/bench_k5w.py [--reps 3] [--jobs 512] [--out FILE]   (one JSON object on stdout, also written to FILE)
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import delly_b200  # noqa: E402
from bench import ClockSampler, gpu_info, host_cores  # noqa: E402
from delly_b200 import synth  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def k5w_batch(n_jobs, seed=1005):
    rng = np.random.default_rng(seed)
    jobs = []
    for i in range(n_jobs):
        m = int(rng.integers(2000, 5001))
        n = int(rng.integers(16400, 40001))
        c, r = synth.wide_consref_job(rng, ("del", "dup", "inv")[i % 3], m, n)
        if rng.random() < 0.1:
            c = synth._ACGT[rng.integers(0, 4, size=m, dtype=np.uint8)]
        jobs.append((c, r))
    return jobs


def host_mem_bytes():
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 8 << 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--jobs", type=int, default=512)
    ap.add_argument("--out")
    a = ap.parse_args()
    jobs = k5w_batch(a.jobs)
    arena, off, ln = synth.pack([x for cr in jobs for x in cr])
    co, cl, ro, rl = off[0::2].copy(), ln[0::2].copy(), off[1::2].copy(), ln[1::2].copy()
    cells = 2 * float(((cl.astype(np.float64) + 1) * (rl.astype(np.float64) + 1)).sum())
    ctx = delly_b200.Context(0)
    ctx.set_profiling(True)
    unsupported = ctx._lib.dgpu_unsupported_count
    unsupported.restype = C.c_uint64
    n0 = int(unsupported(ctx.h))
    sampler = ClockSampler(0)
    sampler.start()
    ks, ts = [], []
    rows = ok = None
    for _ in range(a.reps + 1):   # the first call warms up (module load, workspace)
        t0 = time.perf_counter()
        ok, _, rows = ctx.long_needle(arena, co, cl, ro, rl, max_ref=int(rl.max()))
        ts.append(time.perf_counter() - t0); ks.append(ctx.last_kernel_ms())
    clocks = sampler.stop()
    refused = int(unsupported(ctx.h)) - n0
    assert refused == 0, f"{refused} job(s) refused"
    kms, e2e = float(np.median(ks[1:])), float(np.median(ts[1:]))
    N = len(jobs)
    out = {"gpu": gpu_info(0), "clocks": clocks,
           "family": "K5W longNeedle (lr): consensus 2-5 kb x windows 16.4-40 kb (lnw_kernel, one CTA per alignment)",
           "jobs": N, "cons_len": [int(cl.min()), int(cl.max())], "ref_len": [int(rl.min()), int(rl.max())], "true_results": int(ok.sum()),
           "unit": "alignments/s", "value": N / (kms * 1e-3), "tcups": cells / (kms * 1e-3) / 1e12, "kernel_ms": kms, "kernel_ms_runs": ks[1:],
           "e2e_value": N / e2e}
    R = po.ref()
    if R is not None:
        cores = host_cores()
        per_job = 16 * (5001 * 40001) + (64 << 20)
        threads = max(1, min(cores, int(0.7 * host_mem_bytes()) // per_job))
        cnt = min(N, 2 * threads)
        res = [None] * cnt
        nxt = [0]
        lock = threading.Lock()

        def worker():
            while True:
                with lock:
                    i = nxt[0]; nxt[0] += 1
                if i >= cnt:
                    return
                res[i] = po.long_needle(R, bytes(jobs[i][0]), bytes(jobs[i][1]))

        t0 = time.perf_counter()
        th = [threading.Thread(target=worker) for _ in range(threads)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        dt = time.perf_counter() - t0
        for i in range(cnt):
            eok, e0, e1 = res[i]
            assert bool(ok[i]) == eok and (not eok or rows[i] == (e0, e1)), f"job {i}: GPU alignment differs from the reference"
        out["cpu_baseline"] = {"value": cnt / dt, "unit": "alignments/s", "threads": threads, "cores": cores, "kind": "reference",
                               "sample": f"first {cnt} jobs, {dt:.2f} s, alignments identical to the GPU's"}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
