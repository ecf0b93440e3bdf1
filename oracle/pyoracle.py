"""ctypes loaders for the two CPU checkers (TEST INFRASTRUCTURE ONLY).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module. The product package (delly_b200) never does.

  oracle()  -> oracle/liboracle.so        this repo's CPU restatement (built from oracle/oracle.cpp)
  ref()     -> oracle/_ref/libdelly_ref.so the reference's own sources compiled verbatim
                                           (built in the dev container; travels prebuilt; may be absent)
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = None
_REF = None

u8p = C.POINTER(C.c_uint8)
i32p = C.POINTER(C.c_int32)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)


def build(force=False):
    """Compile liboracle.so (always) and _ref/libdelly_ref.so (only where /root/reference exists)."""
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "oracle.cpp")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"], stdout=subprocess.DEVNULL)
    if os.path.isdir("/root/reference/src"):
        # file targets with dependencies: only what changed is rebuilt (incl. _ref/delly_ref, the reference's drivers against the real htslib)
        subprocess.check_call(["make", "-j8", "-C", _HERE, "ref"], stdout=subprocess.DEVNULL)


def oracle():
    global _ORACLE
    if _ORACLE is None:
        build()
        _ORACLE = C.CDLL(os.path.join(_HERE, "liboracle.so"))
    return _ORACLE


def ref():
    """The compiled reference, or None if it was never built (then tests that need it skip)."""
    global _REF
    if _REF is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF = C.CDLL(p)
    return _REF


_REF2 = None


def ref2():
    """The reference's cluster.h / junction.h compiled verbatim (oracle/_ref/libdelly_ref2.so), or None."""
    global _REF2
    if _REF2 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref2.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF2 = C.CDLL(p)
    return _REF2


_REF3 = None


def ref3():
    """The reference's bolog.h (_computeGLs) and coverage.h (_generateProbes) compiled verbatim (oracle/_ref/libdelly_ref3.so), or None."""
    global _REF3
    if _REF3 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref3.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF3 = C.CDLL(p)
    return _REF3


_REF4 = None


def ref4():
    """The reference's genotype.h (genotypeLR) compiled verbatim over in-memory htslib stand-ins (oracle/_ref/libdelly_ref4.so), or None."""
    global _REF4
    if _REF4 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref4.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF4 = C.CDLL(p)
    return _REF4


_REF5 = None


def ref5():
    """The reference's shortpe.h (assembleSplitReads) compiled verbatim over in-memory htslib stand-ins (oracle/_ref/libdelly_ref5.so), or None."""
    global _REF5
    if _REF5 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref5.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF5 = C.CDLL(p)
    return _REF5


_REF6 = None


def ref6():
    """The reference's util.h compiled itself (getLibraryParams) over in-memory htslib stand-ins (oracle/_ref/libdelly_ref6.so), or None."""
    global _REF6
    if _REF6 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref6.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF6 = C.CDLL(p)
    return _REF6


_REF7 = None


def ref7():
    """The reference's modvcf.h (vcfOutput) compiled verbatim over a recording VCF/BCF stand-in (oracle/_ref/libdelly_ref7.so), or None."""
    global _REF7
    if _REF7 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref7.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF7 = C.CDLL(p)
    return _REF7


_REF8 = None


def ref8():
    """The reference's svanno.h (annotateSV, detectTandemRepeat, the MEI templates) compiled verbatim with its own edlib (oracle/_ref/libdelly_ref8.so), or None."""
    global _REF8
    if _REF8 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref8.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF8 = C.CDLL(p)
    return _REF8


_REF9 = None


def ref9():
    """ref_wrap5.cpp built with the annotation step real and the MM / ML tags visible (the complete long-read chain, oracle/_ref/libdelly_ref9.so), or None."""
    global _REF9
    if _REF9 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref9.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF9 = C.CDLL(p)
    return _REF9


_REF10 = None


def ref10():
    """The sequence-identity helpers of `delly merge` (build-time extract of src/merge.h:187-243) with the reference's edlib (oracle/_ref/libdelly_ref10.so), or None."""
    global _REF10
    if _REF10 is None:
        p = os.path.join(_HERE, "_ref", "libdelly_ref10.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if os.path.exists(p):
            _REF10 = C.CDLL(p)
    return _REF10


def _b(x):
    if isinstance(x, str):
        x = x.encode()
    return x


def _p(a, ty):
    return a.ctypes.data_as(ty)


# ---------------------------------------------------------------- per-item wrappers (lib = oracle() or ref())
def edit_distance(lib, q, t, k=-1, mode=2, task=0, eq=b""):
    """Returns (dist, end0, start0, ops) ; ops only for the reference with task=2."""
    q, t = _b(q), _b(t)
    if lib is _REF:
        d, e, s, nl, al = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
        cap = len(q) + len(t) + 16
        aln = (C.c_ubyte * cap)()
        rc = lib.ref_edlib(q, len(q), t, len(t), k, mode, task, eq, len(eq) // 2, C.byref(d), C.byref(e), C.byref(s),
                           C.byref(nl), aln, cap, C.byref(al))
        assert rc == 0, rc
        return d.value, e.value, s.value, bytes(aln[: al.value])
    e = C.c_int()
    d = lib.ora_edit_distance(q, len(q), t, len(t), k, mode, C.byref(e))
    return d, e.value, None, None


def edit_distance_batch(lib, seqs, q_off, q_len, t_off, t_len, k, mode, threads=1, want_end=False):
    n = len(q_off)
    dist = np.empty(n, np.int32)
    if lib is _REF:
        lib.ref_edlib_distance_batch(_p(seqs, C.c_char_p), _p(q_off.astype(np.uint64), u64p), _p(q_len, u32p),
                                     _p(t_off.astype(np.uint64), u64p), _p(t_len, u32p), _p(k, i32p), mode,
                                     C.c_uint64(n), _p(dist, i32p), threads)
        return dist, None
    end = np.empty(n, np.int32) if want_end else None
    lib.ora_edit_distance_batch(_p(seqs, u8p), _p(q_off, u32p), _p(q_len, u32p), _p(t_off, u32p), _p(t_len, u32p),
                                _p(k, i32p) if k is not None else None, mode, C.c_uint64(n), _p(dist, i32p),
                                _p(end, i32p) if want_end else None, threads)
    return dist, end


def long_needle(lib, s1, s2):
    """Returns (ok, row0, row1)."""
    s1, s2 = _b(s1), _b(s2)
    cap = 2 * (len(s1) + len(s2) + 8)
    rows = C.create_string_buffer(cap)
    L = C.c_int()
    fn = lib.ref_long_needle if lib is _REF else lib.ora_long_needle
    ok = fn(s1, len(s1), s2, len(s2), rows, C.c_long(cap), C.byref(L))
    assert ok >= 0
    if ok == 0:
        return False, b"", b""
    raw = rows.raw
    return True, raw[: L.value], raw[L.value: 2 * L.value]


def longest_homology(lib, s1, s2, thr=-1):
    s1, s2 = _b(s1), _b(s2)
    fn = lib.ref_longest_homology if lib is _REF else lib.ora_longest_homology
    return fn(s1, len(s1), s2, len(s2), thr)


def lcs(lib, a, b):
    a, b = _b(a), _b(b)
    fn = lib.ref_lcs if lib is _REF else lib.ora_lcs
    return fn(a, len(a), b, len(b))


def gotoh(lib, rows1, rows2, sc=(5, -4, -10, -1)):
    """rows1/rows2: lists of equal-length byte strings. Returns (score, merged rows)."""
    r1, r2 = [_b(r) for r in rows1], [_b(r) for r in rows2]
    L1, L2 = len(r1[0]), len(r2[0])
    cap = (len(r1) + len(r2)) * (L1 + L2 + 4)
    out = C.create_string_buffer(cap)
    oL, score = C.c_int(), C.c_int()
    fn = lib.ref_gotoh if lib is _REF else lib.ora_gotoh
    rc = fn(b"".join(r1), len(r1), L1, b"".join(r2), len(r2), L2, sc[0], sc[1], sc[2], sc[3], out, C.c_long(cap),
            C.byref(oL), C.byref(score))
    assert rc == 0
    L = oL.value
    raw = out.raw
    return score.value, [raw[i * L: (i + 1) * L] for i in range(len(r1) + len(r2))]


def consensus(lib, rows, min_clique=2):
    rows = [_b(r) for r in rows]
    L = len(rows[0])
    g, cs, n = C.create_string_buffer(L + 1), C.create_string_buffer(L + 1), C.c_int()
    fn = lib.ref_consensus if lib is _REF else lib.ora_consensus
    fn(b"".join(rows), len(rows), L, min_clique, g, cs, C.byref(n))
    return g.raw[:L], cs.raw[: n.value]


def msa(lib, reads, min_clique=2, sc=(5, -4, -10, -1), want_alignment=False):
    """Returns (nrows, consensus, alignment rows or None)."""
    reads = [_b(r) for r in reads]
    arena = b"".join(reads)
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    tot = int(lens.sum())
    cons = C.create_string_buffer(tot + 16)
    clen, aL = C.c_int(), C.c_int()
    acap = len(reads) * (tot + 16)
    aln = C.create_string_buffer(acap) if want_alignment else None
    fn = lib.ref_msa if lib is _REF else lib.ora_msa
    rows = fn(arena, _p(offs, u32p), _p(lens, u32p), len(reads), min_clique, sc[0], sc[1], sc[2], sc[3], cons, tot + 16,
              C.byref(clen), aln, C.c_long(acap), C.byref(aL))
    assert rows >= 0
    al = None
    if want_alignment:
        L = aL.value
        al = [aln.raw[i * L: (i + 1) * L] for i in range(rows)]
    return rows, cons.raw[: clen.value], al


def msa_nodes(lib, reads, sc=(5, -4, -10, -1)):
    """The guide tree's inner nodes of msa(reads) in creation order, as an int array of rows (R, L, L1, L2, U1, U2): the node's rows and
    alignment columns, its two children's columns (gotoh's DP rows and columns) and their distinct column profiles (0, 0 when both
    children are single reads). Oracle only."""
    reads = [_b(r) for r in reads]
    arena = b"".join(reads)
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    out = np.zeros((max(len(reads), 1), 6), np.int32)
    n = lib.ora_msa_nodes(arena, _p(offs, u32p), _p(lens, u32p), len(reads), sc[0], sc[1], sc[2], sc[3], _p(out, i32p), len(out))
    assert n >= 0
    return out[:n]


def hardware_threads():
    return os.cpu_count() or 1
