#!/usr/bin/env python
"""K1 per kernel class: the configs[1] batch of bench.py (10 M HW edit-distance jobs, probes of 26-80 bp against 150 bp reads) split the
way the library bins it, and each class timed on its own with the one-thread kernels:
  pack W=3 / pack W=5  ed_pack_kernel<3, 1> / <5, 2>: ALT / REF probe pairs of one read (jobs 2i and 2i + 1 on one target) whose two
                       probes fit one column of 3 / 5 words (the library's pack_fits: 33-63 bp with a partner of up to 95 - |q| bp,
                       65-95 bp with up to 159 - |q|, in either order; the benchmark's 33-47 and 65-79 bp pairs),
  nw = 1 / 2 / 3       ed_pair_kernel<NW> for the other pairs whose probes are both of class NW = ceil(|q| / 32), and
                       ed_small_kernel<NW, HW> for the probes whose partner is in another class.
A class's jobs are its pairs first, in batch order (so each pair stays at an even index), then its lone probes.

  kernel_ms           median over the timed calls of the library's CUDA events around the class's kernel (ctx.last_kernel_ms())
  jobs_per_s          jobs of the class / kernel_ms
  thread_columns_per_s  DP columns one thread advances (sum of |t| over the class) / kernel_ms
  window_s            sum of the timed kernel spans: at least --window seconds per class

Every class stays device-resident; the inputs are uploaded once. The card's name, power limit and the SM clock sampled during the timed
calls are part of the record, and so is ctx.int_peak_mix(): the instruction rate of LOP3 chains alone and with IMAD / IMAD.WIDE.U32
chains interleaved, which shows whether the FMA pipe takes IMADs alongside the integer ALU pipe the kernel is bound by.

Usage: python tools/bench_k1.py [--jobs 10000000] [--window 1.2] [--out FILE]   (one JSON line on stdout, also written to FILE)
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import delly_b200  # noqa: E402
from bench import ClockSampler, gpu_info, make_batch  # noqa: E402


def pack_fits(ma, mb, w, wa):
    """edit_distance.cu's pack_fits: A = ma at the bottom of a w-word column with its last row in word wa, B = mb at the top, and at least
    one separator row between them."""
    return (ma > 32 * wa) & (ma <= 32 * wa + 31) & (mb >= 1) & (ma + mb < 32 * w)


def kernels_of(c, n_pair_jobs, n_lone):
    if not isinstance(c, int):
        w = int(c.split("=")[1])
        return [f"ed_pack_kernel<{w}, {(w - 1) // 2}>"]
    return ([f"ed_pair_kernel<{c}>"] if n_pair_jobs else []) + ([f"ed_small_kernel<{c}, HW, false>"] if n_lone else [])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=10_000_000)
    ap.add_argument("--window", type=float, default=1.2, help="seconds of timed kernel work per class")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = delly_b200.Context(0)
    ctx.set_profiling(True)
    b = make_batch(a.jobs, seed=1001)
    nw = (b["q_len"].astype(np.int64) + 31) // 32
    seqs = torch.from_numpy(b["seqs"]).to(dev)
    stream = torch.cuda.current_stream().cuda_stream
    classes = []
    sampler = ClockSampler(0)
    sampler.start()
    q0, q1 = b["q_len"][0::2].astype(np.int64), b["q_len"][1::2].astype(np.int64)
    shared = (b["t_off"][0::2] == b["t_off"][1::2]) & (b["t_len"][0::2] == b["t_len"][1::2])
    pack = {w: shared & (pack_fits(q0, q1, w, wa) | pack_fits(q1, q0, w, wa)) for w, wa in ((3, 1), (5, 2))}
    packed = pack[3] | pack[5]

    def pair_jobs(mask):
        return np.stack([np.nonzero(mask)[0] * 2, np.nonzero(mask)[0] * 2 + 1], axis=1).reshape(-1)

    groups = [(f"pack W={w}", pair_jobs(pack[w]), np.zeros(0, np.int64)) for w in (3, 5)]
    in_pair = np.zeros(len(nw), bool)
    in_pair[pair_jobs(packed | (shared & (nw[0::2] == nw[1::2])))] = True
    for c in (1, 2, 3):
        groups.append((c, pair_jobs(shared & ~packed & (nw[0::2] == c) & (nw[1::2] == c)), np.nonzero((nw == c) & ~in_pair)[0]))
    for c, pairs, lone in groups:
        sel = np.concatenate([pairs, lone])
        if len(sel) == 0:
            continue
        d = {k: torch.from_numpy(np.ascontiguousarray(b[k][sel]).view(np.int32)).to(dev) for k in ("q_off", "q_len", "t_off", "t_len", "k")}
        dist = torch.empty(len(sel), dtype=torch.int32, device=dev)

        def call():
            ctx.edit_distance_dev(seqs, d["q_off"], d["q_len"], d["t_off"], d["t_len"], d["k"], delly_b200.MODE_HW, dist, None, stream)
            torch.cuda.synchronize()
            return ctx.last_kernel_ms()

        for _ in range(3):
            est = call()
        reps = max(10, int(np.ceil(a.window * 1e3 / est)))
        ks = [call() for _ in range(reps)]
        kms = float(np.median(ks))
        cols = int(b["t_len"][sel].astype(np.int64).sum())
        ql = b["q_len"][sel]
        classes.append({"nw" if isinstance(c, int) else "class": c, "kernels": kernels_of(c, len(pairs), len(lone)), "q_len": [int(ql.min()), int(ql.max())], "jobs": int(len(sel)), "paired_jobs": int(len(pairs)), "share": len(sel) / len(nw),
                        "kernel_ms": kms, "kernel_ms_min_max": [float(min(ks)), float(max(ks))], "reps": reps, "window_s": float(sum(ks)) * 1e-3,
                        "jobs_per_s": len(sel) / (kms * 1e-3), "thread_columns_per_s": cols / (kms * 1e-3)})
        del d, dist
    clocks = sampler.stop()
    mix = ctx.int_peak_mix()
    res = {"workload": "configs[1] batch of bench.py split by kernel class: ed_pack_kernel<3, 1> and <5, 2> for the pairs that pack, "
                       "ed_pair_kernel<NW> + ed_small_kernel<NW, HW> per NW = ceil(|q|/32) for the rest",
           "jobs": int(len(nw)), "lib": os.path.relpath(delly_b200.LIB_PATH, ROOT), "gpu": gpu_info(0), "clocks": clocks,
           "int_peak_mix_tera_instr_per_s": mix, "classes": classes}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
