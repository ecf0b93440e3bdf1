#!/usr/bin/env python
"""EPW: edit paths over aligned target slices wider than 16384 columns (dgpu_edit_path_wide).

Workload (seeded): 64 msaWfa-shaped HW paths, reads of 17-40 kb (ONT-like: 4 % substitutions, 3 % insertions, 3 % deletions) against
gapped IUPAC consensus strings of 20-60 kb with the 20 pairs of src/assemble.h:663-693, and 16 unrelated 40 kb NW pairs.

  value        paths/s of the host-pointer calls (both batches, copies in and out included; median of the timed repetitions)
  engines_ms   kernel time per engine in one profiled repetition (torch.profiler, CUDA activities): the distance and start passes
               (ed_*), the band classes (seg_band_kernel), the wavefront classes (seg_kernel), the wide half columns
               (seg_half_wide_kernel) and the wide leaves (seg_leaf_wide_kernel)
  cap_path_s   wall time of one NW path over a slice of DGPU_EP_MAX_SLICE columns (8 % divergence), the figure include/dgpu.h quotes
  cpu_baseline the reference's edlib (oracle/_ref, compiled verbatim) on host threads for the same jobs; every GPU path must equal it

Usage: python tools/bench_ep_wide.py [--reps 3] [--out FILE]   (one JSON object on stdout, also written to FILE)
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import delly_b200  # noqa: E402
from bench import gpu_info, host_cores  # noqa: E402
from delly_b200 import synth  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

IUPAC_EQ = b"MAMCRARGWAWTBAB-SCSGYCYTDCD-KGKTEGE-FTF-"
AMB = np.frombuffer(b"MRWBSYDKEF-N", np.uint8)
ENGINES = ("seg_half_wide_kernel", "seg_leaf_wide_kernel", "seg_band_kernel", "seg_kernel", "ed_", "hb_")


def batches(seed=2049):
    rng = np.random.default_rng(seed)
    hw = []
    for _ in range(64):
        R = int(rng.integers(17_000, 40_001))
        T = int(rng.integers(max(20_000, R + 500), 60_001))
        base = synth._ACGT[rng.integers(0, 4, size=T, dtype=np.uint8)]
        a = int(rng.integers(0, T - R + 1))
        read = synth.mutate_fast(rng, base[a:a + R], sub=0.04, ins=0.03, dele=0.03)
        cons = base.copy()
        k = T // 33
        cons[rng.integers(0, T, size=k)] = AMB[rng.integers(0, len(AMB), size=k)]
        cons = np.insert(cons, np.sort(rng.choice(T, size=T // 30, replace=False)), np.uint8(ord("-")))
        hw += [read, cons]
    nw = []
    for _ in range(16):
        nw += [synth._ACGT[rng.integers(0, 4, size=40_000 - int(rng.integers(0, 600)), dtype=np.uint8)],
               synth._ACGT[rng.integers(0, 4, size=40_000, dtype=np.uint8)]]
    out = []
    for seqs, mode, eq in ((hw, 2, IUPAC_EQ), (nw, 0, b"")):
        arena, off, ln = synth.pack(seqs)
        out.append(dict(seqs=arena, q_off=off[0::2].copy(), q_len=ln[0::2].copy(), t_off=off[1::2].copy(), t_len=ln[1::2].copy(), mode=mode, eq=eq))
    return out


def run(ctx, b):
    return ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["mode"], eq=b["eq"], max_slice=delly_b200.EP_MAX_SLICE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    bs = batches()
    ctx = delly_b200.Context(0)
    res = [run(ctx, b) for b in bs]   # warm-up: module load, workspace
    ts = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        res = [run(ctx, b) for b in bs]
        ts.append(time.perf_counter() - t0)
    npaths = sum(len(b["q_off"]) for b in bs)
    assert all(not r[4].any() for r in res), "a job was refused"
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for b in bs:
            run(ctx, b)
        torch.cuda.synchronize()
    eng = {k: 0.0 for k in ENGINES}
    for ev in prof.key_averages():
        for k in ENGINES:
            if k in ev.key:
                eng[k] += ev.device_time_total / 1e3   # us -> ms
                break
    wall = float(np.median(ts))
    rng = np.random.default_rng(4099)
    t = synth._ACGT[rng.integers(0, 4, size=delly_b200.EP_MAX_SLICE, dtype=np.uint8)]
    q = np.concatenate([t[:32], synth.mutate_fast(rng, t[32:-32], sub=0.048, ins=0.016, dele=0.016), t[-32:]])
    arena, off, ln = synth.pack([q, t])
    cap = dict(seqs=arena, q_off=off[0::2].copy(), q_len=ln[0::2].copy(), t_off=off[1::2].copy(), t_len=ln[1::2].copy(), mode=0, eq=b"")
    t0 = time.perf_counter()
    rc = run(ctx, cap)
    cap_s = time.perf_counter() - t0
    assert rc[4][0] == 0 and int(rc[2][0]) - int(rc[1][0]) + 1 == delly_b200.EP_MAX_SLICE
    out = {"gpu": gpu_info(0),
           "family": "EPW edit paths over slices > 16384 columns: 64 HW reads 17-40 kb vs gapped IUPAC consensus 20-60 kb (20 pairs), "
                     "16 unrelated NW pairs of 40 kb",
           "jobs": npaths, "slices": [int(min(int(e) - int(s) + 1 for r in res for s, e in zip(r[1], r[2]))),
                                      int(max(int(e) - int(s) + 1 for r in res for s, e in zip(r[1], r[2])))],
           "unit": "paths/s", "value": npaths / wall, "wall_s_runs": ts, "engines_ms": {k.rstrip("_"): round(v, 3) for k, v in eng.items()},
           "cap_path_s": round(cap_s, 3), "cap_path": f"one NW pair, {delly_b200.EP_MAX_SLICE} columns, 8 % divergence, distance {int(rc[0][0])}"}
    R = po.ref()
    if R is not None:
        cores = host_cores()
        jobs = [(b, i) for b in bs for i in range(len(b["q_off"]))]

        def one(j):
            b, i = j
            q = b["seqs"][int(b["q_off"][i]):int(b["q_off"][i]) + int(b["q_len"][i])].tobytes()
            t = b["seqs"][int(b["t_off"][i]):int(b["t_off"][i]) + int(b["t_len"][i])].tobytes()
            return po.edit_distance(R, q, t, -1, b["mode"], task=2, eq=b["eq"])

        t0 = time.perf_counter()
        with ThreadPoolExecutor(cores) as ex:
            ref = list(ex.map(one, jobs))
        dt = time.perf_counter() - t0
        k = 0
        for bi, b in enumerate(bs):
            d, st, en, ops, _ = res[bi]
            for i in range(len(b["q_off"])):
                rd, re, rs, rops = ref[k]; k += 1
                assert (int(d[i]), int(st[i]), int(en[i]), ops[i]) == (rd, rs, re, rops), f"batch {bi} job {i}: GPU path differs from the reference"
        out["cpu_baseline"] = {"value": npaths / dt, "unit": "paths/s", "threads": cores, "kind": "reference edlib",
                               "sample": f"all {npaths} jobs, {dt:.2f} s, paths identical to the GPU's"}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
