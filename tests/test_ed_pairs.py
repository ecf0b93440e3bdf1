"""ed_pair_kernel: two HW jobs on one target (jobs 2i and 2i + 1 of a call with equal t_off and t_len and the same one-thread class, no end
locations) run in one thread. Every job's distance matches the oracle's edlib, pairs or not, and so do the reworked last columns of
ed_small_kernel (whole words of four through the fast block) for target lengths of every residue mod 16, in all three modes."""
import os

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALPHA = np.frombuffer(b"ACGT", np.uint8)
ODD = np.frombuffer(b"NRYacgtn-", np.uint8)
TLENS = list(range(1, 41)) + list(range(140, 171)) + [297, 300, 301, 303]


def _cls(ql):
    return (ql + 31) // 32


def _odd(rng, a, rate):
    a = a.copy()
    if len(a) and rng.random() < rate:
        pos = rng.integers(0, len(a), size=int(rng.integers(1, 4)))
        a[pos] = ODD[rng.integers(0, len(ODD), size=len(pos))]
    return a


def _pair_batch(seed):
    """One read and two probes per pair: for every |q| in 1..128 a partner of the same class, targets of every length in TLENS, probes
    cut from the read (with noise) or random, N / IUPAC / lower-case bytes in either probe and in the read (body and last columns)."""
    rng = np.random.default_rng(seed)
    seqs, jobs = [], []   # jobs: (q index, t index)
    for i in range(2 * 128 * 3):
        qa = 1 + i % 128
        c = _cls(qa)
        qb = int(rng.integers(32 * (c - 1) + 1, 32 * c + 1))
        tl = TLENS[int(rng.integers(0, len(TLENS)))]
        t = ALPHA[rng.integers(0, 4, size=tl)]
        qs = []
        for ql in (qa, qb):
            if rng.random() < 0.7 and tl >= ql:
                a0 = int(rng.integers(0, tl - ql + 1))
                q = synth.sub_noise(rng, t[a0:a0 + ql], 0.05)
            else:
                q = ALPHA[rng.integers(0, 4, size=ql)]
            qs.append(_odd(rng, q, 0.2))
        t = _odd(rng, t, 0.3)
        if rng.random() < 0.2:
            t[-min(3, tl):] = ODD[rng.integers(0, len(ODD), size=min(3, tl))]
        ti = len(seqs)
        seqs.append(t)
        for q in qs:
            seqs.append(q)
            jobs.append((len(seqs) - 1, ti))
    arena, off, ln = synth.pack(seqs)
    qi = np.array([j[0] for j in jobs]); ti = np.array([j[1] for j in jobs])
    return dict(seqs=arena, q_off=off[qi].copy(), q_len=ln[qi].copy(), t_off=off[ti].copy(), t_len=ln[ti].copy())


def _unshared(b):
    """The same jobs with every target copied to an offset of its own: nothing pairs."""
    arena = [b["seqs"]]
    t_off = b["t_off"].copy()
    base = len(b["seqs"])
    for i in range(len(t_off)):
        t = b["seqs"][b["t_off"][i]:b["t_off"][i] + b["t_len"][i]]
        arena.append(t)
        t_off[i] = base
        base += len(t)
    return dict(b, seqs=np.concatenate(arena), t_off=t_off)


def _ks(rng, d):
    """Per job: below, at or above the distance, or -1."""
    sel = rng.integers(0, 4, size=len(d))
    return np.where(sel == 0, d - 1, np.where(sel == 1, d, np.where(sel == 2, d + 1, -1))).astype(np.int32)


def _oracle(b, k, mode, want_end=False):
    return po.edit_distance_batch(po.oracle(), b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, mode,
                                  threads=os.cpu_count() or 1, want_end=want_end)


def _pairs(b):
    """Indices i (even) of the jobs that form a pair with i + 1 under ed_slot's rule."""
    n = len(b["q_len"])
    i = np.arange(0, n - 1, 2)
    ca, cb = _cls(b["q_len"][i].astype(np.int64)), _cls(b["q_len"][i + 1].astype(np.int64))
    ok = ((b["t_off"][i] == b["t_off"][i + 1]) & (b["t_len"][i] == b["t_len"][i + 1]) & (b["t_len"][i] > 0) & (ca == cb)
          & (ca >= 1) & (ca <= 4) & (b["q_len"][i] > 0) & (b["q_len"][i + 1] > 0))
    return i[ok]


def test_pair_batch_shape():
    b = _pair_batch(1)
    assert len(_pairs(b)) == len(b["q_len"]) // 2
    assert set(b["q_len"][0::2].tolist()) == set(range(1, 129))
    assert {int(x) % 16 for x in b["t_len"]} == set(range(16))
    assert len(_pairs(_unshared(b))) == 0


@pytest.mark.gpu
def test_pairs_match_oracle_and_unpaired_runs(ctx):
    b = _pair_batch(2)
    d0, _ = _oracle(b, None, 2)
    k = _ks(np.random.default_rng(3), d0)
    d, _ = _oracle(b, k, 2)
    g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, delly_b200.MODE_HW)
    bad = np.nonzero(g != d)[0]
    assert len(bad) == 0, (bad[:5], g[bad[:5]], d[bad[:5]], b["q_len"][bad[:5]], b["t_len"][bad[:5]])
    u = _unshared(b)
    gu = ctx.edit_distance(u["seqs"], u["q_off"], u["q_len"], u["t_off"], u["t_len"], k, delly_b200.MODE_HW)
    assert np.array_equal(gu, g)
    # with end locations nothing pairs either, and the distances are the same
    ge, _ = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, delly_b200.MODE_HW, want_end=True)
    assert np.array_equal(ge, g)


def _mixed_batch(seed):
    """Jobs that must not pair, among pairs that do: equal t_off with another t_len, equal bytes at another offset, a shared target starting
    at an odd job index, members of different classes, |q| = 0 and |q| > 128 members; the batch has an odd length."""
    rng = np.random.default_rng(seed)
    seqs, jobs = [], []

    def add(q, ti, tl=None):
        seqs.append(q)
        jobs.append((len(seqs) - 1, ti, tl))

    def target(tl):
        seqs.append(ALPHA[rng.integers(0, 4, size=tl)])
        return len(seqs) - 1

    def probe(ql):
        return ALPHA[rng.integers(0, 4, size=ql)]

    for r in range(60):
        tl = int(rng.integers(100, 171))
        t = target(tl)
        kind = r % 7
        if kind == 0:    # a real pair
            add(probe(int(rng.integers(33, 65))), t); add(probe(int(rng.integers(33, 65))), t)
        elif kind == 1:  # same t_off, other t_len
            add(probe(40), t); add(probe(50), t, tl - int(rng.integers(1, 5)))
        elif kind == 2:  # the same bytes at another offset
            t2 = len(seqs); seqs.append(seqs[t].copy())
            add(probe(40), t); add(probe(40), t2)
        elif kind == 3:  # a lone job first, so the shared target starts at an odd index; the filler pairs with nothing
            add(probe(30), target(150)); add(probe(70), t); add(probe(75), t)
            add(probe(20), target(120))
        elif kind == 4:  # different classes
            add(probe(32), t); add(probe(33), t)
        elif kind == 5:  # |q| = 0 and |q| > 128
            add(probe(0), t); add(probe(20), t)
            add(probe(129), t); add(probe(100), t)
        else:            # a pair of class 4 and one of class 1
            add(probe(128), t); add(probe(97), t)
            add(probe(1), t); add(probe(32), t)
    add(probe(50), target(150))
    arena, off, ln = synth.pack(seqs)
    qi = np.array([j[0] for j in jobs]); ti = np.array([j[1] for j in jobs])
    tl = np.array([ln[j[1]] if j[2] is None else j[2] for j in jobs], np.uint32)
    b = dict(seqs=arena, q_off=off[qi].copy(), q_len=ln[qi].copy(), t_off=off[ti].copy(), t_len=tl)
    assert len(b["q_len"]) % 2 == 1
    return b


def test_mixed_batch_pairs_only_where_allowed():
    b = _mixed_batch(4)
    p = set(_pairs(b).tolist())
    n = len(b["q_len"])
    assert 0 < len(p) < n // 2
    assert n - 1 not in p and all(i % 2 == 0 for i in p)


@pytest.mark.gpu
def test_mixed_batch_matches_oracle(ctx):
    b = _mixed_batch(5)
    d0, _ = _oracle(b, None, 2)
    k = _ks(np.random.default_rng(6), d0)
    d, _ = _oracle(b, k, 2)
    g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, delly_b200.MODE_HW)
    bad = np.nonzero(g != d)[0]
    assert len(bad) == 0, (bad[:5], g[bad[:5]], d[bad[:5]], b["q_len"][bad[:5]], b["t_len"][bad[:5]])


def _tail_batch(seed):
    """Single jobs for every target length 1..170 and query lengths of every class, with odd bytes in the last columns."""
    rng = np.random.default_rng(seed)
    seqs = []
    for tl in range(1, 171):
        for ql in (int(rng.integers(1, 33)), int(rng.integers(33, 65)), int(rng.integers(65, 97)), int(rng.integers(97, 129))):
            t = ALPHA[rng.integers(0, 4, size=tl)]
            if tl >= ql and rng.random() < 0.6:
                a0 = int(rng.integers(0, tl - ql + 1))
                q = synth.sub_noise(rng, t[a0:a0 + ql], 0.05)
            else:
                q = ALPHA[rng.integers(0, 4, size=ql)]
            q = _odd(rng, q, 0.15)
            t = _odd(rng, t, 0.15)
            if rng.random() < 0.2:
                t[-1] = ODD[rng.integers(0, len(ODD))]
            seqs += [q, t]
    arena, off, ln = synth.pack(seqs)
    return dict(seqs=arena, q_off=off[0::2].copy(), q_len=ln[0::2].copy(), t_off=off[1::2].copy(), t_len=ln[1::2].copy())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("want_end", [True, False])
def test_last_columns_every_target_length(ctx, mode, want_end):
    b = _tail_batch(10 + mode)
    d0, _ = _oracle(b, None, mode)
    k = _ks(np.random.default_rng(20 + mode), d0)
    d, e = _oracle(b, k, mode, want_end=True)
    if want_end:
        g, ge = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, mode, want_end=True)
        ok = d >= 0
        bad = np.nonzero((ge != e) & ok)[0]
        assert len(bad) == 0, (bad[:5], ge[bad[:5]], e[bad[:5]], b["t_len"][bad[:5]])
        assert np.all(ge[~ok] == -1)
    else:
        g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, mode)
    bad = np.nonzero(g != d)[0]
    assert len(bad) == 0, (bad[:5], g[bad[:5]], d[bad[:5]], b["q_len"][bad[:5]], b["t_len"][bad[:5]])


@pytest.mark.gpu
def test_pairs_in_async_device_form(ctx):
    import torch
    b = _pair_batch(7)
    k = _ks(np.random.default_rng(8), _oracle(b, None, 2)[0])
    d, _ = _oracle(b, k, 2)
    dev = torch.device("cuda", 0)
    t = {n: torch.from_numpy(np.ascontiguousarray(b[n]).view(np.int32) if n != "seqs" else b[n]).to(dev)
         for n in ("seqs", "q_off", "q_len", "t_off", "t_len")}
    kt = torch.from_numpy(k).to(dev)
    out = torch.full((len(k),), -7, dtype=torch.int32, device=dev)
    lib = ctx._lib
    assert lib.dgpu_set_async_bound(ctx.h, 256) == 0
    try:
        ctx.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], kt, delly_b200.MODE_HW, out, None, None)
        torch.cuda.synchronize()
    finally:
        lib.dgpu_set_async_bound(ctx.h, 0)
    assert np.array_equal(out.cpu().numpy(), d)


@pytest.mark.gpu
def test_pipelined_host_form_pairs_in_every_range(ctx):
    """3 * 2^18 - 2 jobs in two ranges of an odd size before rounding: the second range still starts on an even job, so ed_pair_kernel runs
    in both; the distances match the oracle."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    n = 3 * (1 << 18) - 2
    b = synth.k1_genotype_batch(n, seed=31)
    assert len(b["q_len"]) == n and len(b["seqs"]) >= 32 << 20
    d, _ = _oracle(b, b["k"], 2)
    # pair classes of each of the two ranges (jobs_per = 393216)
    p = _pairs(b)
    cls = _cls(b["q_len"][p].astype(np.int64))
    want = len(set(cls[p < 393216].tolist())) + len(set(cls[p >= 393216].tolist()))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["k"], delly_b200.MODE_HW)
        torch.cuda.synchronize()
    launches = sum(e.count for e in prof.key_averages() if "ed_pair_kernel" in e.key)
    assert launches == want, (launches, want)
    assert np.array_equal(g, d)
