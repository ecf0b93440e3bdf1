"""msa_kernel (clusters of up to 32 reads) and msa_large_kernel (33 .. 1023 reads) at their internal limits, against the oracle byte for
byte: alignment rows, consensus, n_rows, aln_cols and status of every cluster of each batch.

The cases aim at the Gotoh strip widths (one strip of 4 columns per lane while n + 1 <= 128, then 256-column strips), the 256-bp
bit-parallel LCS, the profile de-duplication (64 distinct column profiles) and the score table's move into the warp's slab
(U1 x U2 > 4096), the 1023-column cap (status 2), the node alignment storage of 32-read clusters with chain-shaped guide trees, the
32/33-read kernel boundary, the arguments (scores, min_clique) and the device forms. The oracle's node export (pyoracle.msa_nodes)
shows that each case reaches the width, profile count or tree it aims at, and decides which status a cluster must get."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po

LCAP = 1023                                     # widest alignment (and longest read) either kernel computes
WIDTHS = (127, 128, 129, 255, 256, 257, 511, 512, 513, 767, 768, 1022, 1023)
SCORES = ((5, -4, -10, -1), (1, -1, -1, -1), (2, -3, -5, -2), (5, -4, 0, 0), (127, -127, -10, -1))
ST_OK, ST_TOO_MANY, ST_TOO_LONG, ST_BAD_CHAR = 0, 1, 2, 3
_BASES = np.frombuffer(b"ACGT", np.uint8)


# ---- cluster generators ----------------------------------------------------------------------------------------------------

def _hap(rng, n):
    return _BASES[rng.integers(0, 4, size=n)]


def _substitute(rng, seq, k, n_frac=0.0):
    """seq with k substitutions at distinct positions (each to another base) and a fraction n_frac of N bases"""
    r = np.array(seq, np.uint8, copy=True)
    k = min(k, len(r))
    pos = rng.choice(len(r), size=k, replace=False)
    r[pos] = _BASES[(np.searchsorted(_BASES, r[pos]) + rng.integers(1, 4, size=k)) % 4]
    if n_frac:
        r[rng.random(len(r)) < n_frac] = ord("N")
    return r.tobytes()


def _family(seed, k, w, sub=0.01):
    """k reads of one w-bp haplotype with ~sub substitutions each: every node of the guide tree is a gap-free w-column alignment"""
    rng = np.random.default_rng(seed)
    hap = _hap(rng, w)
    return [_substitute(rng, hap, int(rng.binomial(w, sub))) for _ in range(k)]


def _ladder(seed, k, length, s):
    """the divergence ladder: read i is one haplotype with i * s substitutions, so the guide tree is (nearly) a chain"""
    rng = np.random.default_rng(seed)
    hap = _hap(rng, length)
    return [_substitute(rng, hap, i * s) for i in range(k)]


def _noisy(seed, k, length, sub, n_frac, jitter=0):
    """k reads of one haplotype with dense substitutions and N bases: many distinct column profiles per node"""
    rng = np.random.default_rng(seed)
    hap = _hap(rng, length + jitter)
    out = []
    for _ in range(k):
        o = int(rng.integers(0, jitter + 1))
        out.append(_substitute(rng, hap[o:o + length], int(rng.binomial(length, sub)), n_frac))
    return out


def _tiling(seed, k, lo, hi, span, err=0.01):
    rng = np.random.default_rng(seed)
    hap = _hap(rng, span)
    out = []
    for _ in range(k):
        L = int(rng.integers(lo, hi + 1))
        s = int(rng.integers(0, span - L + 1))
        out.append(_substitute(rng, hap[s:s + L], int(rng.binomial(L, err))))
    return out


def _batch(clusters):
    reads = [r for c in clusters for r in c]
    coff = np.concatenate([[0], np.cumsum([len(c) for c in clusters])]).astype(np.uint32)
    arena, off, ln = synth.pack(reads) if reads else (np.zeros(1, np.uint8), np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    return dict(seqs=arena, read_off=off, read_len=ln, cluster_off=coff, clusters=clusters)


# ---- expectations ----------------------------------------------------------------------------------------------------------

def _nodes(reads, sc=SCORES[0]):
    return po.msa_nodes(po.oracle(), reads, sc)


def _expected_status(reads, max_reads, sc=SCORES[0]):
    """the status the kernels must give a cluster: 1 above max_reads; 2 for an empty read, a read or a guide-tree node wider than 1023
    columns; 3 for a byte outside ACGTN; else 0"""
    if len(reads) > max_reads:
        return ST_TOO_MANY
    if any(len(r) == 0 or len(r) > LCAP for r in reads):
        return ST_TOO_LONG
    if any(set(r) - set(b"ACGTN") for r in reads):
        return ST_BAD_CHAR
    if len(reads) > 1 and _nodes(reads, sc)[:, 1].max() > LCAP:
        return ST_TOO_LONG
    return ST_OK


def _expected(clusters, mc, sc, max_reads):
    """per cluster: (status, n_rows, consensus, alignment rows) from the oracle, computed in parallel (ctypes releases the GIL)"""
    O = po.oracle()

    def one(reads):
        st = _expected_status(reads, max_reads, sc)
        if st != ST_OK or not reads:
            return st, 0, b"", []
        rows, cs, aln = po.msa(O, reads, mc, sc, want_alignment=True)
        return st, rows, cs, aln

    with ThreadPoolExecutor(max_workers=po.hardware_threads()) as ex:
        return list(ex.map(one, clusters))


def _check(ctx, clusters, mc=2, sc=SCORES[0], max_reads=delly_b200.MSA_LARGE_MAXR, expect=None):
    """run the host form on one batch and compare every cluster with the oracle; returns the outputs"""
    b = _batch(clusters)
    cons, nrows, status, alns = ctx.msa(b["seqs"], b["read_off"], b["read_len"], b["cluster_off"], sc=sc, min_clique=mc,
                                        want_alignment=True, check=False, max_reads=max_reads)
    exp = _expected(clusters, mc, sc, max_reads)
    for i, (st, rows, cs, aln) in enumerate(exp):
        where = (i, len(clusters[i]), sorted({len(r) for r in clusters[i]})[:4], mc, sc)
        assert int(status[i]) == st, where
        assert int(nrows[i]) == rows, where
        assert cons[i] == cs, where
        assert alns[i] == aln, where
    if expect is not None:
        assert [e[0] for e in exp] == list(expect)
    return cons, nrows, status, alns


def _widest(reads):
    return int(_nodes(reads)[:, 1].max())


def _node_bytes(reads):
    """bytes of node alignment storage msa_kernel keeps for the cluster: R x L per node, rounded up to 16"""
    n = _nodes(reads)
    return int(sum((int(r) * int(l) + 15) // 16 * 16 for r, l in n[:, :2]))


# ---- cases -----------------------------------------------------------------------------------------------------------------

def _width_cases(w, large):
    """clusters whose DP runs at w rows x w columns: one-row sides (a read pair, char compare) and profile sides (every other node),
    plus read pairs of w x 64 and 64 x w; 33 reads for msa_large_kernel"""
    if large:
        return [_family(1000 + w, 33, w)]
    rng = np.random.default_rng(2000 + w)
    hap = _hap(rng, w)
    return [_family(3000 + w, 2, w), _family(4000 + w, 6, w),
            [hap.tobytes(), _substitute(rng, hap[:64], 1)], [_substitute(rng, hap[:64], 1), hap.tobytes()]]


def _lcs_cases():
    """read lengths around the 32-bit words and the 256-bp bit vectors of the LCS, mixed <= 256 / > 256 pairs in both positions, and
    all-long clusters (every pair by plain DP)"""
    rng = np.random.default_rng(71)
    hap = _hap(rng, 700)
    sub = lambda a, b: _substitute(rng, hap[a:b], max(1, (b - a) // 100))  # noqa: E731
    lens = (1, 31, 32, 33, 63, 64, 255, 256, 257)
    return [
        [sub(10, 10 + L) for L in lens],
        [sub(0, L) for L in reversed(lens)],
        [sub(0, 300), sub(20, 120)], [sub(20, 120), sub(0, 300)],
        [sub(0, 256), sub(5, 262)], [sub(5, 262), sub(0, 256)],
        [sub(0, 257), sub(3, 260), sub(1, 258)],
        [sub(0, 400), sub(50, 500), sub(100, 357), sub(200, 600)],
        [sub(0, 1), sub(0, 1)], [sub(4, 5), sub(0, 33)],
        [sub(0, 300), sub(40, 296), sub(100, 400), sub(10, 43), sub(60, 320), sub(30, 287)],
    ]


def _ladders():
    """32 reads of 600 and 800 bp (chain-shaped trees that need more node storage than 202,752 bytes), 20-, 31- and 32-read variants"""
    return [_ladder(11, 32, 600, 4), _ladder(12, 32, 800, 5), _ladder(13, 20, 800, 5), _ladder(14, 31, 700, 4), _ladder(15, 32, 400, 3)]


def _profile_cases(large):
    """more than 64 distinct column profiles on a side (the de-duplication overflows); U1 x U2 = 20 x 210, just above the 4096 entries
    of the shared-memory score table; both sides about 1010 columns with more than 64 profiles each (the slab table nearly full).
    Large: 33- and 40-read clusters with overflowing sides (the second has a node wider than 1023 columns), and nodes of 63, 64 and 1023
    rows."""
    if not large:
        return [_noisy(21, 8, 300, 0.15, 0.05), _noisy(131, 8, 70, 0.3, 0.1), _noisy(1, 16, 1005, 0.07, 0.03)]
    return [_noisy(22, 33, 300, 0.15, 0.05), _noisy(23, 40, 120, 0.3, 0.1), _tiling(24, 63, 100, 150, 300), _tiling(25, 64, 100, 150, 300),
            _tiling(26, 1023, 20, 30, 40)]


def _score_cases():
    """clusters for the score sets: tilings, profile-heavy clusters, a width edge and a chain, in both kernels (free gaps, or match and
    mismatch at +-127, widen the last one's alignment beyond 1023 columns)"""
    return [_tiling(31, 12, 100, 150, 260), _tiling(32, 3, 250, 300, 400), _noisy(21, 8, 300, 0.15, 0.05), _family(33, 5, 257),
            _ladder(34, 10, 300, 6), _tiling(81, 33, 100, 150, 300), _noisy(22, 33, 300, 0.15, 0.05)]


# ---- CPU: the oracle is a valid checker for every case ---------------------------------------------------------------------

def _all_cases():
    cl = []
    for w in WIDTHS:
        cl += _width_cases(w, False)
        cl += _width_cases(w, True)
    cl += _lcs_cases() + _ladders() + _profile_cases(False) + _profile_cases(True)
    return cl


def test_oracle_matches_reference_at_msa_edges(ref):
    """the reference's msa compiled verbatim gives the oracle's alignment and consensus for every width, LCS, ladder and profile case,
    and for the score cases at every score set"""
    O = po.oracle()
    cases = _all_cases()
    jobs = [(reads, SCORES[0]) for reads in cases] + [(reads, sc) for reads in _score_cases() for sc in SCORES[1:]]

    def one(job):
        reads, sc = job
        if _expected_status(reads, LCAP, sc) != ST_OK:
            return True
        return po.msa(O, reads, 2, sc, want_alignment=True) == po.msa(ref, reads, 2, sc, want_alignment=True)

    with ThreadPoolExecutor(max_workers=po.hardware_threads()) as ex:
        ok = list(ex.map(one, jobs))
    assert all(ok), [i for i, x in enumerate(ok) if not x]


def test_node_export_reaches_the_aimed_widths():
    """every width case runs its DP at the width it aims at; the ladders are chains that need more than 202,752 bytes of node storage"""
    for w in WIDTHS:
        for reads in _width_cases(w, False)[:2]:
            n = _nodes(reads)
            assert (n[:, 1] == w).all() and (n[:, 2] == w).all() and (n[:, 3] == w).all(), (w, n.tolist())
        for reads in _width_cases(w, False)[2:]:
            n = _nodes(reads)
            assert sorted(n[0, 2:4].tolist()) == [64, w] and n[0, 1] == w
    for reads in _ladders():
        n = _nodes(reads)
        assert n[:, 1].max() <= LCAP
        if len(reads) == 32 and len(reads[0]) >= 600:
            assert _node_bytes(reads) > 202752, _node_bytes(reads)
    assert max(_node_bytes(r) for r in _ladders()) > 202752


def test_node_export_counts_profiles():
    """the export on hand-made clusters: rows, columns, the children's columns and their distinct column profiles"""
    # reads 0 and 1 merge first; then read 2 (A, C, G, A: three profiles) against their two identical rows (four)
    assert _nodes([b"ACGT", b"ACGT", b"ACGA"]).tolist() == [[2, 4, 4, 4, 0, 0], [3, 4, 4, 4, 3, 4]]
    # two pairs of identical rows with nothing in common: one profile per side, the free end gaps put them side by side
    assert _nodes([b"AAAA", b"AAAA", b"CCCC", b"CCCC"]).tolist() == [[2, 4, 4, 4, 0, 0], [2, 4, 4, 4, 0, 0], [4, 8, 4, 4, 1, 1]]
    assert _nodes([b"ACGT"]).shape == (0, 6)


def test_node_export_reaches_the_profile_cases():
    """the profile cases reach what they aim at (U: a side's distinct profiles; more than 64 counts as one per column)"""
    def u(n, k):
        return np.where(n[:, 4 + k] > 64, n[:, 2 + k], n[:, 4 + k])

    over, just, full = (_nodes(r) for r in _profile_cases(False))
    assert (np.maximum(over[:, 4], over[:, 5]) > 64).any()
    prod = u(just, 0) * u(just, 1)
    assert ((prod > 4096) & (prod <= 4300)).any(), just.tolist()
    both = full[(full[:, 4] > 64) & (full[:, 5] > 64)]
    assert len(both) and both[:, 2:4].min() >= 1005 and full[:, 1].max() <= LCAP, full.tolist()
    big = [_nodes(r) for r in _profile_cases(True)]
    assert (np.maximum(big[0][:, 4], big[0][:, 5]) > 64).any()
    assert [int(n[:, 0].max()) for n in big[2:]] == [63, 64, 1023]


# ---- GPU: the kernels against the oracle -----------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("large", [False, True], ids=["msa_kernel", "msa_large_kernel"])
def test_cuda_strip_and_row_edges(ctx, large):
    """DP widths and rows of 127 .. 1023 around the 4-column and 256-column strips, one-row and profile sides"""
    _check(ctx, [c for w in WIDTHS for c in _width_cases(w, large)], expect=[ST_OK] * (len(WIDTHS) * (1 if large else 4)))


@pytest.mark.gpu
def test_cuda_lcs_widths(ctx):
    """reads of 1 .. 257 bp around the LCS words and bit vectors, mixed and all-long pairs; in a 33-read cluster as well"""
    cl = _lcs_cases()
    big = [r for c in cl[:2] + cl[6:8] for r in c]
    big += _tiling(41, 33 - len(big), 250, 300, 500) if len(big) < 33 else []
    _check(ctx, cl + [big], expect=[ST_OK] * (len(cl) + 1))


@pytest.mark.gpu
@pytest.mark.parametrize("large", [False, True], ids=["msa_kernel", "msa_large_kernel"])
def test_cuda_profiles_and_score_table(ctx, large):
    """de-duplication overflow, the score table in the warp's slab (just above 4096 entries and about 1010 x 1010), nodes of 63, 64
    and 1023 rows"""
    cl = _profile_cases(large)
    _check(ctx, cl, expect=[0, 2, 0, 0, 0] if large else [0, 0, 0])


@pytest.mark.gpu
def test_cuda_column_cap(ctx):
    """reads of 1023 bp are computed; a 1024-bp read, or a node wider than 1023 columns, gives status 2 to its cluster alone"""
    rng = np.random.default_rng(51)
    hap = _hap(rng, 1200)
    ok_small, ok_large = _tiling(52, 6, 100, 150, 260), _tiling(53, 40, 100, 150, 260)
    read1024 = [hap[:1024].tobytes(), hap[5:900].tobytes(), hap[10:700].tobytes()]
    wide = [hap[:1000].tobytes(), _substitute(rng, hap[120:1120], 5)]               # one node of 1120 columns
    cl = [ok_small, _family(54, 3, 1023), read1024, ok_small, wide, _ladder(16, 31, 1000, 6), ok_large,
          read1024 + _tiling(55, 30, 100, 150, 260), _family(56, 33, 1023), [hap[:1000].tobytes()] * 2 + _tiling(57, 31, 900, 1000, 1200),
          ok_small]
    assert _widest(wide) > LCAP and _widest(cl[5]) > LCAP and _widest(cl[9]) > LCAP
    _check(ctx, cl, expect=[0, 0, 2, 0, 2, 2, 0, 2, 0, 2, 0])


@pytest.mark.gpu
def test_cuda_chain_trees_fit_node_storage(ctx):
    """ladders of 20 to 32 reads whose chain-shaped guide trees keep up to 293 KB of node alignments are computed like every other cluster
    whose nodes fit 1023 columns"""
    cl = _ladders()
    _check(ctx, cl, expect=[ST_OK] * len(cl), max_reads=32)
    _check(ctx, cl[:2], mc=3, expect=[ST_OK] * 2, max_reads=32)


@pytest.mark.gpu
@pytest.mark.parametrize("max_reads", [32, 33, 1023])
def test_cuda_kernel_boundary(ctx, max_reads):
    """clusters of exactly 32 and 33 reads: 33 reads get status 1 when max_reads is 32, and are computed otherwise"""
    c32, c33 = _tiling(61, 32, 100, 150, 300), _tiling(62, 33, 100, 150, 300)
    cl = [c32, c33, _tiling(63, 5, 100, 150, 200), c33, c32]
    st = [0, 1, 0, 1, 0] if max_reads == 32 else [0] * 5
    _check(ctx, cl, max_reads=max_reads, expect=st)


@pytest.mark.gpu
@pytest.mark.parametrize("mc", [0, 1, 2, 3, 5, 32, 40])
def test_cuda_min_clique(ctx, mc):
    """the coverage threshold max(2, min(min_clique, rows)) on clusters of 2, 5, 32 and 33 reads"""
    cl = [_tiling(71, 2, 100, 150, 200), _tiling(72, 5, 100, 150, 300), _tiling(73, 32, 100, 150, 300), _tiling(74, 33, 100, 150, 300),
          _tiling(75, 40, 80, 150, 400)]
    _check(ctx, cl, mc=mc, expect=[ST_OK] * len(cl))


@pytest.mark.gpu
@pytest.mark.parametrize("sc", SCORES[1:], ids=lambda s: "_".join(map(str, s)))
def test_cuda_scores(ctx, sc):
    """other DnaScores, the int8 table's bound of +-127 included, in both kernels"""
    cl = _score_cases()
    _check(ctx, cl, sc=sc, expect=[0] * 6 + [2 if sc[3] == 0 or sc[0] == 127 else 0])


@pytest.mark.gpu
def test_cuda_score_bound_unsupported(ctx):
    """match or mismatch beyond +-127 does not fit the int8 score table: DGPU_ERR_UNSUPPORTED, nothing computed"""
    b = _batch([_tiling(85, 4, 100, 150, 200)])
    msg = ctx._lib.dgpu_strerror(-5).decode()
    for sc in ((128, -4, -10, -1), (5, -128, -10, -1)):
        with pytest.raises(delly_b200.DgpuError, match=msg):
            ctx.msa(b["seqs"], b["read_off"], b["read_len"], b["cluster_off"], sc=sc)


@pytest.mark.gpu
def test_cuda_bad_reads_fail_alone(ctx):
    """lower-case or IUPAC bytes give status 3, an empty read status 2 (before a bad byte), to their cluster alone, in both kernels"""
    ok = _tiling(91, 6, 100, 150, 200)
    lower = ok[:2] + [ok[2].lower()] + ok[3:]
    iupac = ok[:3] + [ok[3][:50] + b"R" + ok[3][51:]] + ok[4:]
    empty = ok[:3] + [b""] + ok[3:]
    both = [b"", ok[0].lower()] + ok[1:]
    big = _tiling(92, 34, 100, 150, 300)
    cl = [ok, lower, ok, iupac, empty, ok, both, big[:20] + [big[20].lower()] + big[21:], big, big[:10] + [b""] + big[10:], ok]
    _check(ctx, cl, expect=[0, 3, 0, 3, 2, 0, 2, 3, 0, 2, 0])


@pytest.mark.gpu
@pytest.mark.parametrize("max_reads", [32, 1023])
def test_cuda_device_form_on_side_stream(ctx, max_reads):
    """Context.msa_dev on a non-default torch stream, with the alignment dump: byte-identical to the host form"""
    import torch
    cl = [_tiling(101, 5, 100, 150, 200), _tiling(102, 33, 100, 150, 300), _width_cases(257, False)[1], _noisy(21, 8, 300, 0.15, 0.05),
          _tiling(103, 40, 100, 150, 300), _tiling(104, 32, 100, 150, 300), [b"ACGT" * 30]]
    b = _batch(cl)
    cons, nrows, status, alns = ctx.msa(b["seqs"], b["read_off"], b["read_len"], b["cluster_off"], want_alignment=True, check=False,
                                        max_reads=max_reads)
    assert status.tolist() == [0, 1 if max_reads == 32 else 0, 0, 0, 1 if max_reads == 32 else 0, 0, 0]
    ncl = len(cl)
    cap = np.array([sum(len(r) for r in c) for c in cl], np.uint64)
    cons_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.int64)
    acap = np.array([len(c) * 1024 for c in cl], np.int64)
    aln_off = np.concatenate([[0], np.cumsum(acap)[:-1]]).astype(np.int64)
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()  # noqa: E731
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_seqs = dev(b["seqs"], np.uint8)
        d_roff, d_rlen, d_coff = dev(b["read_off"], np.int32), dev(b["read_len"], np.int32), dev(b["cluster_off"], np.int32)
        d_cons = torch.full((int(cap.sum()),), 0xAB, dtype=torch.uint8, device="cuda")
        d_aln = torch.full((int(acap.sum()),), 0xAB, dtype=torch.uint8, device="cuda")
        d_consoff, d_alnoff = dev(cons_off, np.int64), dev(aln_off, np.int64)
        d_clen, d_nrows, d_status, d_acols = (torch.full((ncl,), -1, dtype=torch.int32, device="cuda") for _ in range(4))
        ctx.msa_dev(d_seqs, d_roff, d_rlen, d_coff, ncl, SCORES[0], 2, d_cons, d_consoff, d_clen, d_nrows, d_status,
                    stream=s.cuda_stream, max_reads=max_reads, aln=d_aln, aln_off=d_alnoff, aln_cols=d_acols)
    s.synchronize()
    h_cons, h_aln = d_cons.cpu().numpy(), d_aln.cpu().numpy()
    h_clen, h_nrows, h_status, h_acols = (t.cpu().numpy().view(np.uint32) for t in (d_clen, d_nrows, d_status, d_acols))
    assert h_status.tolist() == status.tolist() and h_nrows.tolist() == nrows.tolist()
    for i in range(ncl):
        assert h_cons[cons_off[i]:cons_off[i] + h_clen[i]].tobytes() == cons[i], i
        L, R = int(h_acols[i]), int(h_nrows[i])
        assert [h_aln[aln_off[i] + r * L:aln_off[i] + (r + 1) * L].tobytes() for r in range(R)] == alns[i], i
        if status[i]:
            assert h_clen[i] == 0 and h_nrows[i] == 0 and h_acols[i] == 0

    # dgpu_msa_dev is the _ex form at max_reads = 32: the 33- and 40-read clusters get status 1
    d_status.fill_(-1)
    rc = ctx._lib.dgpu_msa_dev(ctx.h, C.c_void_p(d_seqs.data_ptr()), C.c_uint64(d_seqs.numel()), C.c_void_p(d_roff.data_ptr()),
                               C.c_void_p(d_rlen.data_ptr()), C.c_void_p(d_coff.data_ptr()), C.c_uint32(ncl), 5, -4, -10, -1, 2,
                               C.c_void_p(d_cons.data_ptr()), C.c_void_p(d_consoff.data_ptr()), C.c_void_p(d_clen.data_ptr()),
                               C.c_void_p(d_nrows.data_ptr()), C.c_void_p(d_status.data_ptr()), None, None, None, C.c_void_p(s.cuda_stream))
    assert rc == 0
    s.synchronize()
    assert d_status.cpu().numpy().view(np.uint32).tolist() == [0, 1, 0, 0, 1, 0, 0]
