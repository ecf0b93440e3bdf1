#!/usr/bin/env python
"""Per-job fixed cost of the K1 one-thread class kernels: the configs[1] batch of bench.py (make_batch) split by class the way
tools/bench_k1.py splits it, each class timed on its own twice, once against its 150 bp reads and once with every target 300 bp long (the
same probes; each read runs on into the bytes after it, and the arena gets 150 random ACGT bytes of tail). The kernel time of a class is
fitted as a + b * columns per job: the intercept a (two points, a = 2 T150 - T300) is what a job costs whatever its target length (job load,
Peq build, launch and tail of the grid), b the cost of one more target column of every job.

  kernel_ms_150 / kernel_ms_300   median ctx.last_kernel_ms() of the class at 150 / 300 bp targets
  fixed_ms, fixed_share           the intercept a, and a / kernel_ms_150
  per_column_ms                   b, per target column of every job of the class

Usage: python tools/k1_fixed_cost.py [--jobs 10000000] [--window 1.0] [--out FILE]   (one JSON line on stdout, also written to FILE)
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import delly_b200  # noqa: E402
from bench import ClockSampler, gpu_info, make_batch  # noqa: E402
from bench_k1 import pack_fits  # noqa: E402


def class_jobs(b):
    """[(name, job indices)]: pack W=3 / W=5 pairs, then the pairs of NW = 1 / 2 / 3 (bench_k1's split, without the lone probes)."""
    nw = (b["q_len"].astype(np.int64) + 31) // 32
    q0, q1 = b["q_len"][0::2].astype(np.int64), b["q_len"][1::2].astype(np.int64)
    shared = (b["t_off"][0::2] == b["t_off"][1::2]) & (b["t_len"][0::2] == b["t_len"][1::2])
    pack = {w: shared & (pack_fits(q0, q1, w, wa) | pack_fits(q1, q0, w, wa)) for w, wa in ((3, 1), (5, 2))}
    packed = pack[3] | pack[5]

    def pair_jobs(mask):
        return np.stack([np.nonzero(mask)[0] * 2, np.nonzero(mask)[0] * 2 + 1], axis=1).reshape(-1)

    out = [(f"pack W={w}", pair_jobs(pack[w])) for w in (3, 5)]
    for c in (1, 2, 3):
        out.append((f"pair NW={c}", pair_jobs(shared & ~packed & (nw[0::2] == c) & (nw[1::2] == c))))
    return [(k, v) for k, v in out if len(v)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=10_000_000)
    ap.add_argument("--window", type=float, default=1.0, help="seconds of timed kernel work per class and target length")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = delly_b200.Context(0)
    ctx.set_profiling(True)
    b = make_batch(a.jobs, seed=1001)
    rng = np.random.default_rng(7)
    tail = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=150)]
    seqs = torch.from_numpy(np.concatenate([b["seqs"], tail])).to(dev)
    stream = torch.cuda.current_stream().cuda_stream
    sampler = ClockSampler(0)
    sampler.start()
    classes, total150, fixed = [], 0.0, 0.0
    for name, sel in class_jobs(b):
        d = {k: torch.from_numpy(np.ascontiguousarray(b[k][sel]).view(np.int32)).to(dev) for k in ("q_off", "q_len", "t_off", "k")}
        dist = torch.empty(len(sel), dtype=torch.int32, device=dev)
        res = {}
        for tl in (150, 300):
            t_len = torch.full((len(sel),), tl, dtype=torch.int32, device=dev)

            def call():
                ctx.edit_distance_dev(seqs, d["q_off"], d["q_len"], d["t_off"], t_len, d["k"], delly_b200.MODE_HW, dist, None, stream)
                torch.cuda.synchronize()
                return ctx.last_kernel_ms()

            for _ in range(3):
                est = call()
            ks = [call() for _ in range(max(10, int(np.ceil(a.window * 1e3 / est))))]
            res[tl] = float(np.median(ks))
        fx = 2 * res[150] - res[300]
        total150 += res[150]
        fixed += fx
        classes.append({"class": name, "jobs": int(len(sel)), "kernel_ms_150": res[150], "kernel_ms_300": res[300], "fixed_ms": fx,
                        "fixed_share": fx / res[150], "per_column_ms": (res[300] - res[150]) / 150})
        del d, dist
    clocks = sampler.stop()
    out = {"workload": "configs[1] batch of bench.py, pair and pack classes timed alone at 150 and 300 bp targets", "jobs": a.jobs,
           "lib": os.path.relpath(delly_b200.LIB_PATH, ROOT), "gpu": gpu_info(0), "clocks": clocks, "classes": classes,
           "sum_kernel_ms_150": total150, "sum_fixed_ms": fixed, "fixed_share_of_sum": fixed / total150}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
