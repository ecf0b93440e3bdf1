#!/usr/bin/env python
"""What the host round trips of dgpu_edit_path[_ex]_dev cost, and what dgpu_set_ep_async_bound saves or adds.

Workloads (all data on the device, one non-default stream, bound = the largest query and target of the workload):
  K4  splitAlign's shape: consensus pieces of 200-1500 bp placed in 2-4 kb SV windows, HW paths, cut into batches of --k4-batch jobs
  K7  msaEdlib rounds: reads of 300-600 bp against a gapped IUPAC consensus of their length, NW paths with the 20 pairs, batches of 32

  sync_ms     the synchronous device form, batch after batch (each call reads its geometry, distances and split rows back)
  async_ms    the same calls under the bound, enqueued back to back (Hirschberg levels planned on the device)
  enqueue_ms  host time until the last async call has returned
  graph_ms    one replay of a CUDA graph holding every async call of the workload
  large       the whole K4 workload in one call: synchronous against asynchronous (bound-shaped launches of kinds that may turn out empty)
  launches    kernel launches of one call of each workload's batch, synchronous and asynchronous

Each figure is the median over --reps repetitions of the whole workload, host clock around work that ends in a stream synchronise. Every
mode's results are compared with the synchronous form's.

Usage: python tools/bench_ep_async.py [--k4-batch 60] [--reps 20] [--out FILE]   (one JSON object on stdout, also written to FILE)
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import delly_b200  # noqa: E402
from bench import gpu_info  # noqa: E402
from delly_b200 import synth  # noqa: E402

ALPHA = np.frombuffer(b"ACGT", np.uint8)
AMB = np.frombuffer(b"MRWBSYDKEF-N", np.uint8)
IUPAC_EQ = b"MAMCRARGWAWTBAB-SCSGYCYTDCD-KGKTEGE-FTF-"   # the 20 pairs of msaEdlib


def sm_clock():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                       timeout=30)
    return float(r.stdout.strip())


def k4_jobs(rng, n):
    seqs = []
    for _ in range(n):
        t = ALPHA[rng.integers(0, 4, size=int(rng.integers(2000, 4000)))]
        a = int(rng.integers(0, len(t) - 1600))
        seqs += [synth.mutate_fast(rng, t[a:a + int(rng.integers(200, 1500))], sub=0.02, ins=0.01, dele=0.01), t]
    return seqs


def k7_jobs(rng, n):
    seqs = []
    for _ in range(n):
        t = ALPHA[rng.integers(0, 4, size=int(rng.integers(300, 600)))]
        c = t.copy()
        k = len(c) // 25
        c[rng.integers(0, len(c), size=k)] = AMB[rng.integers(0, len(AMB), size=k)]
        seqs += [synth.mutate_fast(rng, t, sub=0.03, ins=0.02, dele=0.02), c]
    return seqs


class Batch:
    def __init__(self, seqs, dev):
        import torch
        arena, off, ln = synth.pack(seqs)
        self.q_len_np, self.t_len_np = ln[0::2], ln[1::2]
        self.n = len(self.q_len_np)
        cap = self.q_len_np.astype(np.uint64) + self.t_len_np.astype(np.uint64)
        u32 = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.uint32).view(np.int32)).to(dev)   # noqa: E731
        self.seqs = torch.from_numpy(np.concatenate([arena, np.zeros(64, np.uint8)])).to(dev)
        self.q_off, self.q_len, self.t_off, self.t_len = u32(off[0::2]), u32(ln[0::2]), u32(off[1::2]), u32(ln[1::2])
        self.ops_off = torch.from_numpy(np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64).view(np.int64)).to(dev)
        self.ops = torch.zeros(int(cap.sum()) + 64, dtype=torch.uint8, device=dev)
        self.out = [torch.zeros(self.n, dtype=torch.int32, device=dev) for _ in range(5)]

    def call(self, ctx, mode, eq, s, n, stream):
        d, st, en, ol, stat = self.out
        ctx.edit_path_dev(self.seqs, self.q_off[s:s + n], self.q_len[s:s + n], self.t_off[s:s + n], self.t_len[s:s + n], mode, d[s:s + n],
                          st[s:s + n], en[s:s + n], self.ops, self.ops_off[s:s + n], ol[s:s + n], stat[s:s + n], eq=eq, stream=stream)

    def result(self):
        import torch
        torch.cuda.synchronize()
        return [o.cpu().numpy().copy() for o in self.out] + [self.ops.cpu().numpy().copy()]


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--k4-batch", type=int, default=60)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(2024)
    st = torch.cuda.Stream(device=dev)
    S = st.cuda_stream
    out = {"gpu": gpu_info(0), "reps": a.reps, "unit": "ms per workload (median)"}

    def timed(fn, reps):
        ts, es = [], []
        for _ in range(reps):
            st.synchronize()
            t0 = time.perf_counter()
            fn()
            es.append(time.perf_counter() - t0)
            st.synchronize()
            ts.append(time.perf_counter() - t0)
        return 1e3 * float(np.median(ts)), 1e3 * float(np.median(es))

    def same(x, y):
        return all(np.array_equal(p, q) for p, q in zip(x, y))

    def measure(name, desc, b, mode, eq, bs, large):
        batches = [(s, min(bs, b.n - s)) for s in range(0, b.n, bs)]
        bound = (int(b.q_len_np.max()), int(b.t_len_np.max()))
        ctx = delly_b200.Context(0)

        def workload():
            for s, n in batches:
                b.call(ctx, mode, eq, s, n, S)
        r = {"workload": desc, "batches": len(batches), "bound": list(bound)}
        workload(); want = b.result()
        r["sync_ms"], _ = timed(workload, a.reps)
        l0 = ctx.launches; b.call(ctx, mode, eq, 0, batches[0][1], S); st.synchronize(); r["launches_sync_call"] = ctx.launches - l0
        ctx.set_ep_async_bound(*bound)
        b.ops.fill_(0); workload()
        assert same(b.result(), want), f"{name}: async results differ from the synchronous form's"
        r["async_ms"], r["enqueue_ms"] = timed(workload, a.reps)
        l0 = ctx.launches; b.call(ctx, mode, eq, 0, batches[0][1], S); st.synchronize(); r["launches_async_call"] = ctx.launches - l0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            workload()
        b.ops.fill_(0); torch.cuda.synchronize()
        with torch.cuda.stream(st):
            g.replay()
        assert same(b.result(), want), f"{name}: graph results differ from the synchronous form's"

        def replay():
            with torch.cuda.stream(st):
                g.replay()
        r["graph_ms"], _ = timed(replay, a.reps)
        del g
        if large:
            ctx.set_ep_async_bound(0, 0)
            L = {"jobs": b.n}
            b.call(ctx, mode, eq, 0, b.n, S); want_l = b.result()
            L["sync_ms"], _ = timed(lambda: b.call(ctx, mode, eq, 0, b.n, S), max(3, a.reps // 4))
            ctx.set_ep_async_bound(*bound)
            b.ops.fill_(0); b.call(ctx, mode, eq, 0, b.n, S)
            assert same(b.result(), want_l), f"{name}: async results of the large call differ"
            L["async_ms"], _ = timed(lambda: b.call(ctx, mode, eq, 0, b.n, S), max(3, a.reps // 4))
            r["large"] = L
        ctx.close()
        out[name] = r

    measure("K4", f"splitAlign shape: 1200 HW jobs (consensus 200-1500 bp in 2-4 kb windows) in batches of {a.k4_batch}",
            Batch(k4_jobs(rng, 1200), dev), 2, b"", a.k4_batch, True)
    measure("K7", "msaEdlib rounds: 40 rounds of 32 NW jobs (reads of 300-600 bp against IUPAC consensus, 20 pairs)",
            Batch(k7_jobs(rng, 1280), dev), 0, IUPAC_EQ, 32, False)
    out["sm_clock_mhz_after"] = sm_clock()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
