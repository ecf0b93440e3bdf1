"""Deterministic synthetic workloads of the shapes SURVEY.md §8(d) names (K1..K7).

Everything is generated from numpy's PCG64 with fixed seeds so the GPU path, the oracle and the
compiled reference all see byte-identical inputs. No file IO, no network.
"""
import numpy as np

_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
_COMP = np.zeros(256, np.uint8)
_COMP[:] = np.arange(256, dtype=np.uint8)
for a, b in zip(b"ACGTN", b"TGCAN"):
    _COMP[a] = b


def random_genome(rng, n, n_frac=0.0):
    g = _ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
    if n_frac > 0:
        nruns = max(1, int(n * n_frac / 50))
        for s in rng.integers(0, max(1, n - 50), size=nruns):
            g[s:s + 50] = ord("N")
    return g


def revcomp(a):
    return _COMP[a[::-1]]


def hw_k(qlen, flank_quality=np.float32(0.95)):
    """k exactly as the reference computes it: int(2 * 0.95f * |q|) in float (src/coverage.h:111)."""
    return (np.float32(2) * np.float32(flank_quality) * qlen.astype(np.float32)).astype(np.int32)


def k1_genotype_batch(n_jobs, seed=1001, read_len=150, genome_len=4_000_000, reads_per_site=60, err=0.005):
    """K1: short-read genotyping realignment jobs (src/coverage.h:412-441).

    Each read overlapping a breakpoint yields two HW edit-distance jobs: ALT probe vs read and REF
    probe vs read. Probes are 26..80 bp (2*13 + homology), reads 150 bp; 50 % REF-like reads, 45 %
    ALT-like (carrying the deletion), 5 % unrelated; substitution errors at `err`, and 10 % of the
    reads carry a 1-bp deletion.
    Returns dict(seqs, q_off, q_len, t_off, t_len, k) — numpy arrays, one packed byte arena.
    """
    rng = np.random.default_rng(seed)
    n_reads = (n_jobs + 1) // 2
    n_sites = max(1, n_reads // reads_per_site)
    g = random_genome(rng, genome_len)
    pos = rng.integers(2000, genome_len - 4000, size=n_sites)
    dele = rng.integers(50, 1000, size=n_sites)
    plen = rng.integers(26, 81, size=n_sites)
    half = plen // 2
    # probes: REF = g[p-half : p-half+plen], ALT = g[p-half:p] + g[p+del : p+del+(plen-half)]
    idx = np.arange(80)[None, :]
    ref_idx = (pos - half)[:, None] + idx
    alt_idx = np.where(idx < half[:, None], ref_idx, ref_idx + dele[:, None])
    ref_probe = g[ref_idx]
    alt_probe = g[alt_idx]
    pmask = idx < plen[:, None]
    probe_off_ref = np.concatenate([[0], np.cumsum(plen)[:-1]])
    ref_bytes = ref_probe[pmask]
    alt_bytes = alt_probe[pmask]
    nprobe = int(plen.sum())
    # reads
    site = rng.integers(0, n_sites, size=n_reads)
    kind = rng.random(n_reads)
    start_off = rng.integers(-read_len + 20, -20, size=n_reads)  # read start relative to breakpoint
    ridx = np.arange(read_len + 1, dtype=np.int32)[None, :]
    rstart = (pos[site] + start_off).astype(np.int32)
    base_idx = rstart[:, None] + ridx
    is_alt = (kind >= 0.5) & (kind < 0.95)
    shift = np.where(is_alt[:, None] & (base_idx >= pos[site].astype(np.int32)[:, None]), dele[site].astype(np.int32)[:, None], np.int32(0))
    unrelated = kind >= 0.95
    base_idx += shift
    base_idx = np.where(unrelated[:, None], (rng.integers(0, genome_len - 1, size=n_reads) // 2).astype(np.int32)[:, None] + ridx, base_idx)
    # 1-bp deletion in 10 % of reads: skip one index
    has_del = rng.random(n_reads) < 0.10
    dpos = rng.integers(5, read_len - 5, size=n_reads)
    base_idx += (has_del[:, None] & (ridx >= dpos.astype(np.int32)[:, None]))
    reads = g[base_idx[:, :read_len]]
    # substitution errors: Poisson number of error positions instead of a full-size random mask
    nerr = rng.binomial(reads.size, err)
    epos = rng.integers(0, reads.size, size=nerr)
    reads.reshape(-1)[epos] = _ACGT[rng.integers(0, 4, size=nerr, dtype=np.uint8)]
    seqs = np.concatenate([ref_bytes, alt_bytes, reads.reshape(-1)]).astype(np.uint8)
    read_off = 2 * nprobe + np.arange(n_reads, dtype=np.int64) * read_len
    # jobs: (ALT probe, read), (REF probe, read) interleaved like process_batch's two calls per job
    q_off = np.empty(2 * n_reads, np.int64)
    q_off[0::2] = nprobe + probe_off_ref[site]
    q_off[1::2] = probe_off_ref[site]
    q_len = np.repeat(plen[site], 2)
    t_off = np.repeat(read_off, 2)
    t_len = np.full(2 * n_reads, read_len)
    q_off, q_len, t_off, t_len = q_off[:n_jobs], q_len[:n_jobs], t_off[:n_jobs], t_len[:n_jobs]
    out = dict(seqs=seqs, q_off=q_off.astype(np.uint32), q_len=q_len.astype(np.uint32), t_off=t_off.astype(np.uint32),
               t_len=t_len.astype(np.uint32))
    out["k"] = hw_k(out["q_len"])
    return out


def mutate(rng, s, sub=0.0, ins=0.0, dele=0.0):
    """Per-base substitution/insertion/deletion noise on a uint8 array (python loop: small inputs only)."""
    out = []
    for ch in s:
        r = rng.random()
        if r < dele:
            continue
        if r < dele + sub:
            out.append(_ACGT[rng.integers(0, 4)])
            continue
        out.append(ch)
        if r < dele + sub + ins:
            out.append(_ACGT[rng.integers(0, 4)])
    return np.array(out, dtype=np.uint8)


def pack(seqs):
    """Pack a list of uint8 arrays / bytes into (arena, off[uint32], len[uint32])."""
    arrs = [np.frombuffer(s, np.uint8) if isinstance(s, (bytes, bytearray)) else np.asarray(s, np.uint8) for s in seqs]
    lens = np.array([len(a) for a in arrs], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens.astype(np.int64))[:-1]]).astype(np.uint32) if len(arrs) else np.zeros(0, np.uint32)
    arena = np.concatenate(arrs).astype(np.uint8) if len(arrs) and lens.sum() else np.zeros(0, np.uint8)
    return arena, offs, lens


def mutate_fast(rng, s, sub=0.0, ins=0.0, dele=0.0):
    """Vectorised per-base substitution / insertion / deletion noise (same model as mutate(), different random stream)."""
    s = np.asarray(s, np.uint8)
    r = rng.random(len(s))
    out = s.copy()
    is_sub = (r >= dele) & (r < dele + sub)
    out[is_sub] = _ACGT[rng.integers(0, 4, size=int(is_sub.sum()), dtype=np.uint8)]
    cnt = np.ones(len(s), np.int64)
    cnt[r < dele] = 0
    is_ins = (r >= dele + sub) & (r < dele + sub + ins)
    cnt[is_ins] = 2
    res = np.repeat(out, cnt)
    # the second copy of an inserted position becomes a random base
    ends = np.cumsum(cnt)[is_ins] - 1
    res[ends] = _ACGT[rng.integers(0, 4, size=len(ends), dtype=np.uint8)]
    return res


def sub_noise(rng, a, rate):
    """Vectorised substitution noise (fast path for large synthetic batches)."""
    a = a.copy()
    k = rng.binomial(len(a), rate) if len(a) else 0
    if k:
        a[rng.integers(0, len(a), size=k)] = _ACGT[rng.integers(0, 4, size=k, dtype=np.uint8)]
    return a


def _revcomp(a):
    """reverse complement of an ACGT array"""
    a = np.asarray(a, np.uint8)
    out = a[::-1].copy()
    for x, y in zip(b"ACGT", b"TGCA"):
        out[a[::-1] == x] = y
    return out


def wide_consref_job(rng, kind, m, n, bp=None, noise=0.02):
    """One consensus / window pair shaped like _getSVRef's output (src/split.h:114-160) for a window of n columns and a consensus of about
    m bases. 'del': one window, flank + deleted segment + flank, the consensus joins the two flanks (breakpoint at column bp of the window);
    'dup' / 'inv': two flanks of n/2 columns cut around the two breakpoints, taken from distant places of the genome (the second one
    reverse-complemented for 'inv'); the consensus joins the first flank's left part to the second flank's right part."""
    g = _ACGT[rng.integers(0, 4, size=2 * n + 100, dtype=np.uint8)]
    h = m // 2
    if kind == "del":
        ref = g[:n]
        a = bp if bp is not None else m
        b = n - (m - h) - int(rng.integers(0, max(1, (n - a - m) // 4)))
        cons = np.concatenate([ref[a - h:a], ref[b:b + (m - h)]])
    else:
        half = n // 2
        second = g[n + 50:n + 50 + (n - half)]
        ref = np.concatenate([g[:half], _revcomp(second) if kind == "inv" else second])
        p = bp if bp is not None else half // 2 + int(rng.integers(0, half // 4))
        q = half + (n - half) // 2
        cons = np.concatenate([ref[p - h:p], ref[q:q + (m - h)]])
    return sub_noise(rng, cons, noise), ref


def k3_consref_batch(n_jobs, seed=1003, cons_range=(150, 300), err=0.01, kinds=(0, 1, 2, 3), ref_cap=None, genome_len=2_000_000,
                     fast=False):
    """K3/K5: consensus vs SV-reference-window jobs shaped like _getSVRef's output (src/split.h:70-163).

    For every job a breakpoint pair is planted in a random genome and the window the reference would
    cut for it (two flanks of up to |cons| bp around each breakpoint, one of them reverse-complemented
    for inversion-type SVs) is paired with a consensus spanning the junction (length in cons_range,
    substitution/indel noise `err`). ~10 % of the jobs get an unrelated consensus (longNeedle -> false).
    Returns dict(seqs, c_off, c_len, r_off, r_len, svt).
    """
    rng = np.random.default_rng(seed)
    g = random_genome(rng, genome_len)
    seqs = []
    svts = []
    for _ in range(n_jobs):
        svt = int(rng.choice(kinds))
        L = int(rng.integers(cons_range[0], cons_range[1] + 1))
        p1 = int(rng.integers(20000, genome_len - 40000))
        size = int(rng.integers(L + 50, 5000))
        p2 = p1 + size
        b = L  # boundary = consensus size (src/split.h:655)
        lo1, hi1 = p1 - b, min(p1 + b, (p1 + p2) // 2)
        lo2, hi2 = max((p1 + p2) // 2 + 1, p2 - b), p2 + b
        left, right = g[lo1:hi1], g[lo2:hi2]
        off = int(rng.integers(L // 4, 3 * L // 4))
        if svt == 2:      # deletion: left flank + right flank
            ref = np.concatenate([left, right])
            cons = np.concatenate([g[p1 - off:p1], g[p2:p2 + (L - off)]])
        elif svt == 3:    # duplication: right window first
            ref = np.concatenate([right, left])
            cons = np.concatenate([g[p2 - off:p2], g[p1:p1 + (L - off)]])
        elif svt == 0:    # 3to3 inversion: left + revcomp(right)
            ref = np.concatenate([left, revcomp(right)])
            cons = np.concatenate([g[p1 - off:p1], revcomp(g[p2 - (L - off):p2])])
        else:             # 5to5 inversion: revcomp(left) + right
            ref = np.concatenate([revcomp(left), right])
            cons = np.concatenate([revcomp(g[p1:p1 + off]), g[p2:p2 + (L - off)]])
        if rng.random() < 0.10:
            cons = _ACGT[rng.integers(0, 4, size=L, dtype=np.uint8)]
        elif err > 0:
            cons = sub_noise(rng, cons, err) if fast else mutate(rng, cons, sub=err / 2, ins=err / 4, dele=err / 4)
        if ref_cap is not None:
            ref = ref[:ref_cap]
        seqs += [cons, ref]
        svts.append(svt)
    arena, off, ln = pack(seqs)
    return dict(seqs=arena, c_off=off[0::2].copy(), c_len=ln[0::2].copy(), r_off=off[1::2].copy(), r_len=ln[1::2].copy(),
                svt=np.array(svts, np.int32))


def k2_msa_batch(n_clusters, seed=1002, read_len=150, nreads=(2, 20), max_off=120, err=0.005, genome_len=1_000_000, fast=False):
    """K2: split-read clusters for msa() — n ~ U[nreads] reads of read_len bp tiling a planted deletion
    breakpoint with start offsets U[-max_off, +max_off] around (breakpoint - read_len/2), substitution /
    indel noise `err`. Returns dict(seqs, read_off, read_len, cluster_off)."""
    rng = np.random.default_rng(seed)
    g = random_genome(rng, genome_len)
    reads = []
    coff = [0]
    for _ in range(n_clusters):
        n = int(rng.integers(nreads[0], nreads[1] + 1))
        p = int(rng.integers(5000, genome_len - 10000))
        dele = int(rng.integers(50, 2000))
        hap = np.concatenate([g[p - 2 * read_len - max_off:p], g[p + dele:p + dele + 2 * read_len + max_off]])
        bp = 2 * read_len + max_off
        for _ in range(n):
            st = bp - read_len // 2 + int(rng.integers(-max_off, max_off + 1))
            r = hap[st:st + read_len]
            if err > 0:
                r = sub_noise(rng, r, err) if fast else mutate(rng, r, sub=err * 0.6, ins=err * 0.2, dele=err * 0.2)
            reads.append(r)
        coff.append(len(reads))
    arena, off, ln = pack(reads)
    return dict(seqs=arena, read_off=off, read_len=ln, cluster_off=np.array(coff, np.uint32))
