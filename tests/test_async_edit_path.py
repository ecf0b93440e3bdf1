"""The asynchronous edit-path device forms (include/dgpu.h: dgpu_set_ep_async_bound).

Under a bound the edit-path forms plan every Hirschberg level on the device and read nothing back. Checked here: results byte-identical to
the synchronous forms and to the reference's edlib over the batches of the edit-path suites (imported from them), calls that return while
the device is still busy, a splitAlign-shaped and an msaEdlib-shaped chain captured into CUDA graphs and replayed on new data (two contexts),
refusals of jobs beyond the bound, and the synchronous forms unchanged after switching back."""
import ctypes as C
import os
import re
import time

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from test_edit_path import _jobs, _long_jobs
from test_edit_path_long import IUPAC_EQ, _check_paths, _depth_lb, _packed, _rand, _shared_arena, _slice_batch
from test_edit_path_wide import CAP, _check, _mixed_batch, _nw_batch, _tall_batch, _wide_shared_arena

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_setter_is_declared_and_exported():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dgpu.h")).read(), flags=re.S)
    assert re.search(r"\bint\s+dgpu_set_ep_async_bound\s*\(dgpu_ctx\*\s*ctx,\s*uint32_t\s+\w+,\s*uint32_t\s+\w+\)", txt)
    assert hasattr(delly_b200.lib(), "dgpu_set_ep_async_bound")
    assert hasattr(delly_b200.Context, "set_ep_async_bound")


@pytest.fixture
def fresh():
    """Contexts of their own (a bound holds workspace until its context closes)."""
    ctxs = []

    def make():
        ctxs.append(delly_b200.Context(0))
        return ctxs[-1]
    yield make
    for c in ctxs:
        c.close()


def _empty_jobs():
    """Empty queries, empty targets and both empty, between ordinary jobs."""
    rng = np.random.default_rng(77)
    seqs = []
    for ql, tl in ((0, 50), (40, 0), (0, 0), (30, 90), (0, 1), (1, 0), (64, 64)):
        seqs += [_rand(rng, ql), _rand(rng, tl)]
    return _packed(seqs)


def _deep_batch():
    """Problems of about 16 kb on both sides with ACG repeats: at least five levels of recursion, ties deciding at every level."""
    acg = lambda n: np.resize(np.frombuffer(b"ACG", np.uint8), n)   # noqa: E731
    rng = np.random.default_rng(1250)
    t = _rand(rng, 16200)
    return _packed([acg(16000), acg(16384), synth.mutate_fast(rng, t, sub=0.05, ins=0.02, dele=0.02)[:16200], t])


# name: (batch, mode, eq, max_slice of the wide form or None, expected status or None)
CASES = {
    "short_nw": (lambda: _jobs(11, 300, 64, 64, 0), 0, b"", None, None),
    "short_shw": (lambda: _jobs(12, 300, 150, 300, 1), 1, b"", None, None),
    "short_hw_iupac": (lambda: _jobs(13, 300, 60, 120, 2), 2, IUPAC_EQ, None, None),
    "split_nw": (lambda: _long_jobs(14, 12, 3000, 7000, 0, 0.05), 0, b"", None, None),
    "split_hw": (lambda: _long_jobs(15, 12, 3000, 9000, 2, 0.05), 2, b"", None, None),
    "split_nw_iupac": (lambda: _long_jobs(16, 12, 3000, 7000, 0, 0.05), 0, IUPAC_EQ, None, None),
    "slices_nw_iupac": (lambda: _slice_batch(0, IUPAC_EQ), 0, IUPAC_EQ, None, None),
    "slices_shw": (lambda: _slice_batch(1, b""), 1, b"", None, None),
    "slices_hw": (lambda: _slice_batch(2, b""), 2, b"", None, None),
    "deep": (_deep_batch, 0, b"", None, None),
    "shared_arena_hw": (lambda: _shared_arena(b""), 2, b"", None, None),
    "shared_arena_nw_iupac": (lambda: _shared_arena(IUPAC_EQ), 0, IUPAC_EQ, None, None),
    "empty": (_empty_jobs, 2, b"", None, None),
    "wide_nw": (lambda: _nw_batch(b"", 3400), 0, b"", CAP, None),
    "wide_mixed": (lambda: _mixed_batch(3600)[0], 0, b"", CAP, None),
    "wide_mixed_classic": (lambda: _mixed_batch(3600)[0], 0, b"", None, "wide"),
    "wide_shared_arena_hw": (lambda: _wide_shared_arena(3500), 2, b"", CAP, None),
    "tall": (lambda: _tall_batch(3950), 0, b"", CAP, None),
    "tall_max_slice": (lambda: _tall_batch(3950), 0, b"", 16384, [0, 2]),
}


def _run(ctx, b, mode, eq, max_slice):
    return ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], mode, eq=eq, max_slice=max_slice)


def _same(x, y):
    return all(np.array_equal(a, c) for a, c in zip(x[:3], y[:3])) and x[3] == y[3] and np.array_equal(x[4], y[4])


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_bound_matches_synchronous_form_and_reference(fresh, ref, case):
    """Under a bound exactly at the batch's largest job (so the deepest level the bound admits is reached), every output equals the
    synchronous form's byte for byte and the reference's edlib."""
    make, mode, eq, max_slice, status = CASES[case]
    b = make()
    sync, bound = fresh(), fresh()
    want = _run(sync, b, mode, eq, max_slice)
    bound.set_ep_async_bound(max(1, int(b["q_len"].max())), max(1, int(b["t_len"].max())))
    if status == "wide":
        status = [2 if w else 0 for w in _mixed_batch(3600)[1]]
    if case == "empty":
        pass   # edlib returns before any location exists for these; the synchronous form's start = -1 convention is the yardstick
    elif max_slice is None:
        _check_paths(bound, ref, b, mode, eq, status)
    else:
        _check(bound, ref, b, mode, eq, max_slice, status)
    got = _run(bound, b, mode, eq, max_slice)
    assert _same(got, want)
    if case == "empty":
        assert not got[4].any() and got[3] == want[3]
    if case == "deep":
        assert min(_depth_lb(int(q), int(t)) for q, t in zip(b["q_len"], b["t_len"])) >= 5


# ---------------------------------------------------------------------------------------------------------------------------------------
class _Dev:
    """One edit-path batch in device memory, with its output buffers."""

    def __init__(self, b, dev):
        import torch
        self.b, self.n = b, len(b["q_off"])
        cap = b["q_len"].astype(np.uint64) + b["t_len"].astype(np.uint64)
        self.ops_off_np = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
        u32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).to(dev)   # noqa: E731
        arena = np.zeros((len(b["seqs"]) + 64 + 15) // 16 * 16, np.uint8)
        arena[:len(b["seqs"])] = b["seqs"]
        self.seqs = torch.from_numpy(arena).to(dev)
        self.q_off, self.q_len, self.t_off, self.t_len = (u32(b[k]) for k in ("q_off", "q_len", "t_off", "t_len"))
        self.ops_off = torch.from_numpy(self.ops_off_np.view(np.int64)).to(dev)
        self.ops = torch.zeros(int(cap.sum()) + 64, dtype=torch.uint8, device=dev)
        self.out = [torch.zeros(self.n, dtype=torch.int32, device=dev) for _ in range(5)]   # dist, start, end, ops_len, status

    def load(self, b):
        """New sequences of the same shape, in the same buffers."""
        import torch
        assert all(np.array_equal(b[k], self.b[k]) for k in ("q_off", "q_len", "t_off", "t_len"))
        self.b = b
        self.seqs[:len(b["seqs"])].copy_(torch.from_numpy(b["seqs"]))

    def call(self, ctx, mode, eq=b"", stream=None):
        d, s, e, ol, st = self.out
        ctx.edit_path_dev(self.seqs, self.q_off, self.q_len, self.t_off, self.t_len, mode, d, s, e, self.ops, self.ops_off, ol, st, eq=eq,
                          stream=stream)

    def clear(self):
        self.ops.fill_(0x55)
        for o in self.out:
            o.fill_(-7)

    def result(self):
        import torch
        torch.cuda.synchronize()
        d, s, e, ol, st = (o.cpu().numpy().copy() for o in self.out)
        o = self.ops.cpu().numpy()
        return d, s, e, [o[int(a):int(a) + int(n)].tobytes() for a, n in zip(self.ops_off_np, ol)], st.view(np.uint32)


def _split_align(seed):
    """splitAlign's shape: consensus pieces of 200-1500 bases placed in 2-4 kb windows (HW), and prefixes against the windows (SHW)."""
    rng = np.random.default_rng(seed)
    seqs = []
    for _ in range(24):
        t = _rand(rng, int(rng.integers(2000, 4000)))
        a = int(rng.integers(0, len(t) - 1600))
        seqs += [synth.mutate_fast(rng, t[a:a + int(rng.integers(200, 1500))], sub=0.02, ins=0.01, dele=0.01), t]
    return _packed(seqs)


def _msa_round(seed):
    """An msaEdlib round: reads of 300-600 bases against a gapped IUPAC consensus of their length (NW, the 20 pairs)."""
    rng = np.random.default_rng(seed)
    amb = np.frombuffer(b"MRWBSYDKEF-N", np.uint8)
    seqs = []
    for _ in range(32):
        t = _rand(rng, int(rng.integers(300, 600)))
        c = t.copy()
        k = len(c) // 25
        c[rng.integers(0, len(c), size=k)] = amb[rng.integers(0, len(amb), size=k)]
        seqs += [synth.mutate_fast(rng, t, sub=0.03, ins=0.02, dele=0.02), c]
    return _packed(seqs)


def _same_shape(b, seed):
    """The batch b with new random bytes in every sequence (same offsets and lengths)."""
    nb = dict(b)
    nb["seqs"] = _rand(np.random.default_rng(seed), len(b["seqs"]))
    return nb


@pytest.mark.gpu
def test_bounded_call_returns_before_the_stream_runs(fresh):
    """Behind a one-second device sleep on its stream, a bounded call (HW with splits) returns long before the sleep ends; after a
    synchronise its results are the synchronous form's."""
    import torch
    dev = torch.device("cuda", 0)
    b = _long_jobs(21, 8, 3000, 6000, 2, 0.05)
    ctx = fresh()
    d = _Dev(b, dev)
    d.clear(); d.call(ctx, 2)
    want = d.result()
    ctx.set_ep_async_bound(int(b["q_len"].max()), int(b["t_len"].max()))
    st = torch.cuda.Stream(device=dev)
    d.call(ctx, 2, stream=st.cuda_stream)   # warm-up: the per-job scratch
    torch.cuda.synchronize()
    d.clear()
    torch.cuda.synchronize()
    ev = torch.cuda.Event()
    with torch.cuda.stream(st):
        torch.cuda._sleep(2_000_000_000)   # about a second
    t0 = time.perf_counter()
    d.call(ctx, 2, stream=st.cuda_stream)
    dt = time.perf_counter() - t0
    with torch.cuda.stream(st):
        ev.record()
    pending = not ev.query()
    torch.cuda.synchronize()
    assert pending and dt < 0.2, (pending, dt)
    assert _same(d.result(), want)


@pytest.mark.gpu
def test_chains_captured_into_graphs(fresh):
    """On two contexts: a splitAlign-shaped chain (HW and SHW paths, then longNeedle under its bound) and an msaEdlib round (NW distances,
    then NW paths with the 20 pairs) captured into CUDA graphs, replayed on new bytes in the same buffers; the results equal the
    synchronous calls'."""
    import torch
    from test_async_device_forms import _Dev as _LnDev, _sr_jobs
    dev = torch.device("cuda", 0)
    ctxs = [fresh(), fresh()]
    chains = []
    for k, ctx in enumerate(ctxs):
        sa, mr = _split_align(31 + k), _msa_round(41 + k)
        ln = _LnDev(_sr_jobs(40, seed=51 + k), dev)
        c = dict(hw=_Dev(sa, dev), shw=_Dev(sa, dev), msa=_Dev(mr, dev), ln=ln,
                 ed=torch.zeros(len(mr["q_off"]), dtype=torch.int32, device=dev))
        qmax = max(int(sa["q_len"].max()), int(mr["q_len"].max()))
        tmax = max(int(sa["t_len"].max()), int(mr["t_len"].max()))
        ctx.set_ep_async_bound(qmax, tmax)
        assert delly_b200.lib().dgpu_set_async_bound(ctx.h, C.c_uint32(max(qmax, tmax))) == 0
        ctx.set_ln_async_bound(400, 4000)
        chains.append(c)

    def run(ctx, c, stream):
        c["hw"].call(ctx, 2, stream=stream)
        c["shw"].call(ctx, 1, stream=stream)
        ln = c["ln"]
        ctx.long_needle_dev(ln.seqs, ln.c_off, ln.c_len, ln.r_off, ln.r_len, ln.aln, ln.aln_off, ln.aln_len, ln.ok, ln.info, stream=stream)
        m = c["msa"]
        ctx.edit_distance_dev(m.seqs, m.q_off, m.q_len, m.t_off, m.t_len, None, 0, c["ed"], stream=stream)
        m.call(ctx, 0, eq=IUPAC_EQ, stream=stream)

    def results(c):
        torch.cuda.synchronize()
        return [c[k].result() for k in ("hw", "shw", "msa")] + [c["ln"].result(), c["ed"].cpu().numpy().copy()]

    side = torch.cuda.Stream(device=dev)
    graphs = []
    for ctx, c in zip(ctxs, chains):
        torch.cuda.synchronize()
        run(ctx, c, side.cuda_stream)   # warm-up: the per-job scratch
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run(ctx, c, torch.cuda.current_stream().cuda_stream)
        graphs.append(g)
    for k, c in enumerate(chains):
        for name, seed in (("hw", 61), ("shw", 61), ("msa", 71)):
            c[name].load(_same_shape(c[name].b, seed + k))
        for d in (c["hw"], c["shw"], c["msa"]):
            d.clear()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for g in graphs:
            g.replay()
    got = [results(c) for c in chains]
    sync = fresh()
    for c, r in zip(chains, got):
        for d in (c["hw"], c["shw"], c["msa"]):
            d.clear()
        torch.cuda.synchronize()
        run(sync, c, side.cuda_stream)
        want = results(c)
        for x, y in zip(r[:3], want[:3]):
            assert _same(x, y) and not x[4].any()
        assert all(np.array_equal(x, y) for x, y in zip(r[3], want[3]))
        assert np.array_equal(r[4], want[4])


@pytest.mark.gpu
def test_refusals_under_the_bound(fresh):
    """Jobs beyond max_query or max_target get status 4 alone (dist = start = end = -1, no ops); their neighbours equal the synchronous
    form's, and dgpu_unsupported_count rises by exactly their number once the work has finished."""
    import torch
    dev = torch.device("cuda", 0)
    b = _long_jobs(23, 10, 2000, 5000, 2, 0.05)
    qm, tm = int(np.sort(b["q_len"])[-3]), int(np.sort(b["t_len"])[-3])
    over = (b["q_len"] > qm) | (b["t_len"] > tm)
    assert 2 <= over.sum() < len(over)
    sync, ctx = fresh(), fresh()
    want = _run(sync, b, 2, b"", None)
    ctx.set_ep_async_bound(qm, tm)
    before = ctx.unsupported
    d = _Dev(b, dev)
    d.clear(); d.call(ctx, 2)
    got = d.result()
    assert ctx.unsupported == before + int(over.sum())
    for i in range(len(over)):
        if over[i]:
            assert (got[0][i], got[1][i], got[2][i], got[3][i], got[4][i]) == (-1, -1, -1, b"", 4), i
        else:
            assert (got[0][i], got[1][i], got[2][i], got[3][i], got[4][i]) == (want[0][i], want[1][i], want[2][i], want[3][i], 0), i


@pytest.mark.gpu
def test_switching_back_and_setter_arguments(fresh):
    """After (0, 0) a call makes the launches of a fresh context and gives its outputs; arguments out of range are DGPU_ERR_ARG."""
    b = _long_jobs(25, 6, 3000, 6000, 0, 0.05)
    a, c = fresh(), fresh()
    a.set_ep_async_bound(int(b["q_len"].max()), int(b["t_len"].max()))
    bounded = _run(a, b, 0, IUPAC_EQ, None)
    a.set_ep_async_bound(0, 0)
    _run(c, b, 0, IUPAC_EQ, None)   # first calls may reserve; compare the second
    l0, l1 = a.launches, c.launches
    x, y = _run(a, b, 0, IUPAC_EQ, None), _run(c, b, 0, IUPAC_EQ, None)
    assert a.launches - l0 == c.launches - l1
    assert _same(x, y) and _same(bounded, y)
    for q, t in ((0, 5), (5, 0), (CAP + 1, 5), (5, CAP + 1)):
        with pytest.raises(delly_b200.DgpuError):
            a.set_ep_async_bound(q, t)
