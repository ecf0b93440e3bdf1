#!/usr/bin/env python
"""What the host round trip of dgpu_long_needle_dev costs, and what dgpu_set_ln_async_bound saves or adds.

Workload: the K3 batch of bench.py (4096 consensus of 150-300 bp against SV windows of 600-1600 bp), cut into batches of --batch jobs, the
size alignConsensusBatch sees per SV batch. All data on the device; one non-default stream; bound = the largest consensus and window.

  sync_ms     the synchronous device form, batch after batch (each call reads its class counts back and plans on the host)
  async_ms    the same calls under the bound, enqueued back to back (device-side planning, no readback)
  enqueue_ms  host time until the last async call has returned (the device is still working)
  graph_ms    one replay of a CUDA graph holding every async call of the workload
  large       the whole K3 call of bench.py (49,152 jobs in one call): synchronous against asynchronous, which launches every class the
              bound admits at its full grid (the CTAs of classes that turn out empty return at once)

Each figure is the median over --reps repetitions of the whole workload, host clock around work that ends in a stream synchronise. Every
mode's results are compared with the synchronous form's.

Usage: python tools/bench_ln_async.py [--batch 300] [--reps 20] [--out FILE]   (one JSON object on stdout, also written to FILE)
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


def sm_clock():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                       timeout=30)
    return float(r.stdout.strip())


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=300)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    b = synth.k3_consref_batch(4096, seed=1003, cons_range=(150, 300), err=0.01, fast=True)
    rep = 12   # bench.py's K3 call
    c_off, c_len = np.tile(b["c_off"], rep), np.tile(b["c_len"], rep)
    r_off, r_len = np.tile(b["r_off"], rep), np.tile(b["r_len"], rep)
    N = len(c_off)
    cap = c_len.astype(np.uint64) + r_len.astype(np.uint64)
    aln_off = np.concatenate([[0], np.cumsum(2 * cap)[:-1]]).astype(np.uint64)
    u32 = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.uint32).view(np.int32)).to(dev)   # noqa: E731
    T = dict(seqs=torch.from_numpy(np.concatenate([b["seqs"], np.zeros(64, np.uint8)])).to(dev), c_off=u32(c_off), c_len=u32(c_len),
             r_off=u32(r_off), r_len=u32(r_len), aln_off=torch.from_numpy(aln_off.view(np.int64)).to(dev))
    aln = torch.zeros(int(2 * cap.sum()) + 64, dtype=torch.uint8, device=dev)
    alen = torch.zeros(N, dtype=torch.int32, device=dev)
    ok = torch.zeros(N, dtype=torch.uint8, device=dev)
    n4 = len(b["c_off"])
    batches = [(s, min(a.batch, n4 - s)) for s in range(0, n4, a.batch)]   # the 4096 unique jobs
    bound = (int(c_len.max()), int(r_len.max()))
    ctx = delly_b200.Context(0)
    st = torch.cuda.Stream(device=dev)
    S = st.cuda_stream

    def call(s, n):
        ctx.long_needle_dev(T["seqs"], T["c_off"][s:s + n], T["c_len"][s:s + n], T["r_off"][s:s + n], T["r_len"][s:s + n], aln,
                            T["aln_off"][s:s + n], alen[s:s + n], ok[s:s + n], stream=S)

    def workload():
        for s, n in batches:
            call(s, n)

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

    def result(n):
        torch.cuda.synchronize()
        return ok[:n].cpu().numpy().copy(), alen[:n].cpu().numpy().copy(), aln.cpu().numpy().copy()

    def same(x, y):
        return all(np.array_equal(p, q) for p, q in zip(x, y))

    out = {"gpu": gpu_info(0), "workload": f"K3: {n4} jobs (consensus 150-300 bp, windows 600-1600 bp) in batches of {a.batch}",
           "batches": len(batches), "bound": list(bound), "reps": a.reps, "unit": "ms per workload (median)"}
    # synchronous device form
    workload(); want = result(n4)
    out["sync_ms"], _ = timed(workload, a.reps)
    # asynchronous: back to back, then one graph of all calls
    ctx.set_ln_async_bound(*bound)
    aln.fill_(0); workload(); got = result(n4)
    assert same(got, want), "async results differ from the synchronous form's"
    out["async_ms"], out["enqueue_ms"] = timed(workload, a.reps)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        workload()
    aln.fill_(0); torch.cuda.synchronize()
    with torch.cuda.stream(st):
        g.replay()
    assert same(result(n4), want), "graph results differ from the synchronous form's"

    def replay():
        with torch.cuda.stream(st):
            g.replay()
    out["graph_ms"], _ = timed(replay, a.reps)
    out["launches_per_async_call"] = None
    l0 = ctx.launches; call(0, batches[0][1]); st.synchronize(); out["launches_per_async_call"] = ctx.launches - l0
    # the whole K3 call, bound-shaped launches against exact ones
    ctx.set_ln_async_bound(0, 0)
    l0 = ctx.launches; call(0, N); st.synchronize(); out["launches_per_sync_large_call"] = ctx.launches - l0
    want_l = result(N)
    large = {"jobs": N}
    large["sync_ms"], _ = timed(lambda: call(0, N), max(3, a.reps // 4))
    ctx.set_ln_async_bound(*bound)
    aln.fill_(0); call(0, N)
    assert same(result(N), want_l), "async results of the large call differ"
    large["async_ms"], _ = timed(lambda: call(0, N), max(3, a.reps // 4))
    out["large"] = large
    out["sm_clock_mhz_after"] = sm_clock()
    ctx.set_ln_async_bound(0, 0)
    ctx.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
