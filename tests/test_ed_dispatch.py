"""Edit-distance dispatch: ed_count_kernel classifies every job once (its count slot kept as one byte, class starts written by its last block),
ed_scatter_kernel places the jobs from those bytes, and the class kernels run side by side on the context's fork/join streams, joined back
into the caller's stream. Every job's result matches the oracle's edlib on batches that reach every class, in the host form, the device form
on a non-default stream and the asynchronous device form; a caller that synchronises only its own stream sees finished results; class
kernels overlap in time; every non-empty class is launched once."""
import os
import re

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po

ALPHA = np.frombuffer(b"ACGT", np.uint8)
ODD = np.frombuffer(b"NRYacgtn-", np.uint8)
MODES = {"hw": (delly_b200.MODE_HW, False), "shw_end": (delly_b200.MODE_SHW, True), "nw": (delly_b200.MODE_NW, False)}


def _cls(ql, tl):
    return 0 if ql == 0 or tl == 0 else (ql + 31) // 32 if ql <= 128 else 5


def _pack_fits(ma, mb, w, wa):
    return 32 * wa < ma <= 32 * wa + 31 and mb >= 1 and ma + mb < 32 * w


def _pack_class(m0, m1):
    for cls, (w, wa) in ((10, (3, 1)), (11, (5, 2))):
        if _pack_fits(m0, m1, w, wa) or _pack_fits(m1, m0, w, wa):
            return cls
    return -1


def _slots(b, pair):
    """ed_slot of every job: 0 trivial, 1..4 one thread, 5 one warp, 5 + c pairs of class c, 10 / 11 packs, -1 the odd member of a pair."""
    ql, tl, to = b["q_len"].astype(int), b["t_len"].astype(int), b["t_off"].astype(int)
    n = len(ql)
    out = []
    for i in range(n):
        c = _cls(ql[i], tl[i])
        o = i ^ 1
        if not pair or not 1 <= c <= 4 or o >= n or to[o] != to[i] or tl[o] != tl[i]:
            out.append(c)
            continue
        pk = _pack_class(ql[o], ql[i]) if i & 1 else _pack_class(ql[i], ql[o])
        if pk >= 0:
            out.append(-1 if i & 1 else pk)
        elif _cls(ql[o], tl[i]) != c:
            out.append(c)
        else:
            out.append(-1 if i & 1 else 5 + c)
    return np.array(out)


def _odd(rng, a, rate):
    a = a.copy()
    if len(a) and rng.random() < rate:
        pos = rng.integers(0, len(a), size=int(rng.integers(1, 4)))
        a[pos] = ODD[rng.integers(0, len(ODD), size=len(pos))]
    return a


def _mixed_batch(seed, mode, bound=None):
    """Jobs in units of two (jobs 2i, 2i + 1), every sequence at most `bound` bytes: lone probes of every one-thread class and one-warp
    queries on targets of their own, target-sharing pairs of one class that do not pack, pairs that pack into 3 or 5 words, empty queries and
    targets, N / IUPAC / lower-case bytes. NW queries are the target with substitutions and indels, so that band passes certify most long
    jobs; without a bound a few queries pass 2048 rows (multi-stripe)."""
    rng = np.random.default_rng(seed)
    cap = bound or 10 ** 9
    seqs, jobs = [], []

    def target(tl):
        seqs.append(_odd(rng, ALPHA[rng.integers(0, 4, size=tl)], 0.3))
        return len(seqs) - 1

    def query(ti, ql):
        t = seqs[ti]
        if mode == delly_b200.MODE_NW and ql > 0 and rng.random() < 0.8:
            q = synth.mutate_fast(rng, t, sub=0.03, ins=0.02, dele=0.02)[:min(cap, max(ql, 1))]
        elif rng.random() < 0.7 and len(t) >= ql:
            a0 = int(rng.integers(0, len(t) - ql + 1))
            q = synth.sub_noise(rng, t[a0:a0 + ql], 0.05)
        else:
            q = ALPHA[rng.integers(0, 4, size=ql)]
        seqs.append(_odd(rng, q, 0.2))
        jobs.append((len(seqs) - 1, ti))

    def tlen(ql):
        if mode == delly_b200.MODE_NW and rng.random() < 0.8:
            return int(min(cap, max(1, ql + rng.integers(-ql // 10 - 1, ql // 10 + 2))))
        return int(rng.integers(1, min(cap, 300) + 1))

    def lone(ql):
        query(target(tlen(ql)), ql)

    def shared(m0, m1):
        ti = target(tlen(max(m0, m1)))
        query(ti, m0)
        query(ti, m1)

    ones = [m for m in range(1, 129) if m <= cap]
    for m in ones:                                    # lone probes of classes 1..4, two per unit on different targets
        lone(m)
        lone(int(rng.choice(ones)))
    for c in range(1, 5):                             # pairs of one class that do not pack
        lo, hi = 32 * (c - 1) + 1, min(32 * c, cap)
        got = 0
        while lo <= hi and got < 40:
            m0, m1 = int(rng.integers(lo, hi + 1)), int(rng.integers(lo, hi + 1))
            if _pack_class(m0, m1) < 0:
                shared(m0, m1)
                got += 1
    for _ in range(60):                               # pairs that pack, in both job orders
        for w, wa in ((3, 1), (5, 2)):
            ma = int(rng.integers(32 * wa + 1, 32 * wa + 32))
            mb = int(rng.integers(1, 32 * w - ma))
            if max(ma, mb) <= cap:
                if rng.random() < 0.5:
                    ma, mb = mb, ma
                shared(ma, mb)
    if cap > 128:                                     # one warp per job, band passes in NW
        for _ in range(40):
            lone(int(rng.integers(129, min(cap, 1500) + 1)))
            lone(int(rng.integers(129, min(cap, 400) + 1)))
    if cap > 2048:
        for ql in (2100, 2600):
            lone(ql)
            lone(int(rng.integers(1, 129)))
    for _ in range(4):                                # trivial jobs: empty query, empty target
        query(target(int(rng.integers(1, min(cap, 60) + 1))), 0)
        seqs.append(np.zeros(0, np.uint8))
        query(len(seqs) - 1, int(rng.integers(1, min(cap, 60) + 1)))
    arena, off, ln = synth.pack(seqs)
    qi = np.array([j[0] for j in jobs])
    ti = np.array([j[1] for j in jobs])
    b = dict(seqs=arena, q_off=off[qi].copy(), q_len=ln[qi].copy(), t_off=off[ti].copy(), t_len=ln[ti].copy())
    assert len(b["q_len"]) % 2 == 0 and max(b["q_len"].max(), b["t_len"].max()) <= cap
    return b


def _ks(rng, d):
    sel = rng.integers(0, 4, size=len(d))
    return np.where(sel == 0, d - 1, np.where(sel == 1, d, np.where(sel == 2, d + 1, -1))).astype(np.int32)


def _oracle(b, k, mode, want_end=False):
    return po.edit_distance_batch(po.oracle(), b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, mode,
                                  threads=os.cpu_count() or 1, want_end=want_end)


def _dev(b, k, dev):
    import torch
    t = {n: torch.from_numpy(np.ascontiguousarray(b[n]).view(np.int32)).to(dev) for n in ("q_off", "q_len", "t_off", "t_len")}
    t["seqs"] = torch.from_numpy(np.concatenate([b["seqs"], np.zeros(64, np.uint8)])).to(dev)[:len(b["seqs"])]
    t["k"] = torch.from_numpy(k).to(dev)
    return t


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("bound", [None, 64, 256])
def test_mixed_batch_reaches_every_class(mode, bound):
    m, _ = MODES[mode]
    b = _mixed_batch(1, m, bound)
    s = _slots(b, pair=mode == "hw")
    want = set(range(1, 5 if bound != 64 else 3))
    if mode == "hw":
        want |= {5 + c for c in want} | {10} | ({11} if bound != 64 else set())
    if bound != 64:
        want.add(5)
    assert want <= set(s.tolist()) and 0 in s
    if bound is None:
        assert b["q_len"].max() > 2048


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", ["host", "dev_stream", "async64", "async256"])
def test_every_class_matches_oracle(ctx, mode, form):
    import torch
    m, want_end = MODES[mode]
    bound = {"async64": 64, "async256": 256}.get(form)
    b = _mixed_batch(2 + (bound or 0), m, bound)
    k = _ks(np.random.default_rng(3), _oracle(b, None, m)[0])
    d, e = _oracle(b, k, m, want_end)
    if form == "host":
        g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, m, want_end=want_end)
        gd, ge = g if want_end else (g, None)
    else:
        dev = torch.device("cuda", 0)
        t = _dev(b, k, dev)
        n = len(k)
        out = torch.full((n,), -7, dtype=torch.int32, device=dev)
        end = torch.full((n,), -7, dtype=torch.int32, device=dev) if want_end else None
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream())
        if bound:
            assert ctx._lib.dgpu_set_async_bound(ctx.h, bound) == 0
        try:
            ctx.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], t["k"], m, out, end, s.cuda_stream)
        finally:
            ctx._lib.dgpu_set_async_bound(ctx.h, 0)
        s.synchronize()
        gd = out.cpu().numpy()
        ge = end.cpu().numpy() if want_end else None
    bad = np.nonzero(gd != d)[0]
    assert len(bad) == 0, (bad[:5], gd[bad[:5]], d[bad[:5]], b["q_len"][bad[:5]], b["t_len"][bad[:5]])
    if want_end:
        assert np.array_equal(ge, e)


@pytest.mark.gpu
def test_caller_stream_sync_sees_finished_results(ctx):
    """Two calls on two caller streams; each result is read after synchronising only the stream it was launched on. The class kernels run on
    the context's pool streams, so this holds only if each call joins them back into its caller's stream."""
    import torch
    dev = torch.device("cuda", 0)
    bs = [synth.k1_genotype_batch(200_000, seed=s) for s in (41, 42)]
    ds = [_oracle(b, b["k"], delly_b200.MODE_HW)[0] for b in bs]
    ts = [_dev(b, b["k"], dev) for b in bs]
    outs = [torch.full((len(b["k"]),), -7, dtype=torch.int32, device=dev) for b in bs]
    s1, s2 = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    s1.wait_stream(torch.cuda.current_stream())
    assert ctx._lib.dgpu_set_async_bound(ctx.h, 256) == 0
    try:
        t = ts[0]
        ctx.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], t["k"], delly_b200.MODE_HW, outs[0], None, s1.cuda_stream)
        s2.wait_stream(s1)   # the context's scratch is shared: the second call follows the first on the device
        t = ts[1]
        ctx.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], t["k"], delly_b200.MODE_HW, outs[1], None, s2.cuda_stream)
    finally:
        ctx._lib.dgpu_set_async_bound(ctx.h, 0)
    s2.synchronize()
    g2 = outs[1].cpu().numpy()
    s1.synchronize()
    g1 = outs[0].cpu().numpy()
    assert np.array_equal(g1, ds[0])
    assert np.array_equal(g2, ds[1])


def _kernels(prof):
    """(kernel name, template arguments, start us, end us) of every ed_* class kernel in a profile."""
    out = []
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        mt = re.search(r"(ed_\w+_kernel)(?:<([^>]*)>)?", e.name)
        if mt:
            out.append((mt.group(1), (mt.group(2) or "").replace(" ", ""), e.time_range.start, e.time_range.end))
    return out


@pytest.mark.gpu
def test_class_kernels_overlap():
    """A K1 batch in the host form: only its non-empty classes are launched, and at least two of them run at the same time."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    b = synth.k1_genotype_batch(400_000, seed=43)
    c = delly_b200.Context(0)
    try:
        c.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["k"], delly_b200.MODE_HW)   # pool streams, scratch
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            g = c.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["k"], delly_b200.MODE_HW)
            torch.cuda.synchronize()
    finally:
        c.close()
    assert np.array_equal(g, _oracle(b, b["k"], delly_b200.MODE_HW)[0])
    ks = [x for x in _kernels(prof) if x[0] in ("ed_small_kernel", "ed_pair_kernel", "ed_pack_kernel")]
    assert len(ks) >= 3, ks
    overlaps = [(a[:2], z[:2]) for i, a in enumerate(ks) for z in ks[i + 1:] if a[2] < z[3] and z[2] < a[3]]
    assert overlaps, ks


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_each_nonempty_class_launches_once(ctx, mode):
    import torch
    from torch.profiler import ProfilerActivity, profile
    m, want_end = MODES[mode]
    b = _mixed_batch(5, m)
    s = _slots(b, pair=mode == "hw" and not want_end)
    kern = {5: ("ed_long_kernel", f"{m},false"), 10: ("ed_pack_kernel", "3,1"), 11: ("ed_pack_kernel", "5,2")}
    for c in range(1, 5):
        kern[c] = ("ed_small_kernel", f"{c},{m},{'true' if want_end else 'false'}")
        kern[5 + c] = ("ed_pair_kernel", str(c))
    want = sorted(kern[c] for c in set(s.tolist()) if c > 0)
    assert len(want) >= (11 if mode == "hw" else 5)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], None, m, want_end=want_end)
        torch.cuda.synchronize()
    ks = _kernels(prof)
    got = sorted((x[0], x[1]) for x in ks if x[0] in ("ed_small_kernel", "ed_pair_kernel", "ed_pack_kernel", "ed_long_kernel"))
    assert got == want
    assert [x[0] for x in ks].count("ed_count_kernel") == 1 and [x[0] for x in ks].count("ed_scatter_kernel") == 1
    assert not any(x[0] == "ed_offsets_kernel" for x in ks)


@pytest.mark.gpu
def test_async_form_captures_into_a_graph():
    """The asynchronous device form, fork and join onto the pool streams included, can be captured into a CUDA graph once its scratch and
    its streams exist (include/dgpu.h, dgpu_set_async_bound)."""
    import torch
    dev = torch.device("cuda", 0)
    b = synth.k1_genotype_batch(100_000, seed=44)
    d = _oracle(b, b["k"], delly_b200.MODE_HW)[0]
    t = _dev(b, b["k"], dev)
    out = torch.full((len(d),), -7, dtype=torch.int32, device=dev)
    c = delly_b200.Context(0)
    try:
        assert c._lib.dgpu_set_async_bound(c.h, 256) == 0

        def call():
            c.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], t["k"], delly_b200.MODE_HW, out, None,
                                torch.cuda.current_stream().cuda_stream)

        call()   # the scratch slots and the pool streams
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call()
        out.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        got = out.cpu().numpy()
    finally:
        c.close()
    assert np.array_equal(got, d)
