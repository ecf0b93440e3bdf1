#!/usr/bin/env python
"""K2L: split-read consensus of clusters with more than 32 reads (translocations, `-p` above 32), the workload of msa_large_kernel,
next to K2 (2-20 reads per cluster, msa_kernel) measured the same way in the same process.

  value       clusters/s from the library's CUDA events around the MSA kernels (median of the timed repetitions)
  e2e_value   clusters/s of the host-pointer call (copies in and out included)
  cpu_baseline  the reference's msa (oracle/_ref, compiled verbatim) on all host cores, on the first clusters of the batch; the GPU
                consensus of those clusters must equal the reference's

Usage: python tools/bench_k2l.py [--reps 3] [--out FILE]   (one JSON object on stdout, also written to FILE)
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import delly_b200  # noqa: E402
from bench import gpu_info, host_cores  # noqa: E402
from delly_b200 import synth  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def family(ctx, name, b, max_reads, reps, ref_clusters):
    N = len(b["cluster_off"]) - 1
    ks, ts = [], []
    cons = None
    for i in range(reps + 1):   # the first call warms up (module load, workspace)
        t0 = time.perf_counter()
        cons, _, _ = ctx.msa(b["seqs"], b["read_off"], b["read_len"], b["cluster_off"], max_reads=max_reads)
        ts.append(time.perf_counter() - t0); ks.append(ctx.last_kernel_ms())
    kms, e2e = float(np.median(ks[1:])), float(np.median(ts[1:]))
    nr = np.diff(b["cluster_off"].astype(np.int64))
    out = {"family": name, "jobs": N, "reads_per_cluster": [int(nr.min()), int(nr.max()), round(float(nr.mean()), 1)], "unit": "clusters/s",
           "value": N / (kms * 1e-3), "kernel_ms": kms, "kernel_ms_runs": ks[1:], "e2e_value": N / e2e}
    R = po.ref()
    if R is not None:
        cores = host_cores()
        cnt = min(N, ref_clusters * cores)
        co = b["cluster_off"]
        csum = np.concatenate([[0], np.cumsum(b["read_len"].astype(np.uint64))])
        cap = csum[co[1:cnt + 1]] - csum[co[:cnt]]
        cons_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
        cbuf = np.zeros(int(cap.sum()), np.uint8); clen = np.zeros(cnt, np.uint32)
        ro64 = b["read_off"].astype(np.uint64)
        t0 = time.perf_counter()
        R.ref_msa_batch(C.c_char_p(b["seqs"].ctypes.data), C.c_void_p(ro64.ctypes.data), C.c_void_p(b["read_len"].ctypes.data),
                        C.c_void_p(co.ctypes.data), C.c_uint32(cnt), 2, 5, -4, -10, -1, C.c_char_p(cbuf.ctypes.data),
                        C.c_void_p(cons_off.ctypes.data), C.c_void_p(clen.ctypes.data), cores)
        dt = time.perf_counter() - t0
        for i in range(cnt):
            assert cons[i] == cbuf[int(cons_off[i]):int(cons_off[i]) + int(clen[i])].tobytes(), f"{name}: GPU consensus differs from the reference"
        out["cpu_baseline"] = {"value": cnt / dt, "unit": "clusters/s", "cores": cores, "kind": "reference",
                               "sample": f"first {cnt} clusters, {dt:.2f} s, consensus identical to the GPU's"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = delly_b200.Context(0)
    ctx.set_profiling(True)
    res = {"gpu": gpu_info(0), "families": [
        family(ctx, "K2L msa (sr): 33-300 reads x 150 bp per cluster (msa_large_kernel, one CTA per cluster)",
               synth.k2_msa_batch(264, seed=1004, nreads=(33, 300), fast=True), 300, a.reps, 2),   # two waves of one CTA per SM
        family(ctx, "K2 msa (sr): 2-20 reads x 150 bp per cluster (msa_kernel, one warp per cluster)",
               synth.k2_msa_batch(8192, seed=1002, fast=True), 32, a.reps, 8),
    ]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
