"""delly_b200 — H100-native (sm_90a) batched realignment kernels for Delly's split-read path.

This Python package is only the thin ctypes face of the C ABI in include/dgpu.h (used by tests and
bench.py). The product is libdelly_b200.so (hand-written CUDA, delly_b200/csrc) plus the C++ host
mirror of the reference's interface in delly_b200/host. There is no CPU fallback: loading fails
loudly when the library has not been built, and Context() fails when no H100 is visible.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DGPU_LIB") or os.path.join(_HERE, "libdelly_b200.so")   # DGPU_LIB: development aid (kernel variants under variants/)

MODE_NW, MODE_SHW, MODE_HW = 0, 1, 2
MSA_LARGE_MAXR = 1023   # DGPU_MSA_LARGE_MAXR: the largest cluster Context.msa(max_reads=...) can compute
LN_MAX_REF = 65535      # DGPU_LN_MAX_REF: the widest reference window Context.long_needle(max_ref=...) can compute
EP_MAX_SLICE = 262144   # DGPU_EP_MAX_SLICE: the widest aligned target slice Context.edit_path(max_slice=...) can trace

_lib = None


class DgpuError(RuntimeError):
    pass


def lib():
    """Load libdelly_b200.so (built in-tree by build.sh / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DgpuError(
                f"{LIB_PATH} is missing: run ./build.sh (nvcc, sm_90a). delly_b200 has no CPU fallback.")
        _lib = C.CDLL(LIB_PATH)
        _lib.dgpu_last_error.restype = C.c_char_p
        _lib.dgpu_strerror.restype = C.c_char_p
        _lib.dgpu_launch_count.restype = C.c_uint64
        _lib.dgpu_last_kernel_ms.restype = C.c_float
    return _lib


HOST_LIB_PATH = os.path.join(_HERE, "libdelly_b200_host.so")
_hostlib = None


def hostlib():
    """The C++ host mirror of the reference interface (delly_b200/host) with its flat test hooks."""
    global _hostlib
    if _hostlib is None:
        lib()  # the CUDA library first (RPATH $ORIGIN also finds it)
        if not os.path.exists(HOST_LIB_PATH):
            raise DgpuError(f"{HOST_LIB_PATH} is missing: run ./build.sh")
        _hostlib = C.CDLL(HOST_LIB_PATH)
    return _hostlib


def _ptr(x):
    """Raw address of a numpy array / torch tensor / int / None as c_void_p."""
    if x is None:
        return C.c_void_p(0)
    if isinstance(x, np.ndarray):
        assert x.flags["C_CONTIGUOUS"]
        return C.c_void_p(x.ctypes.data)
    if hasattr(x, "data_ptr"):
        assert x.is_contiguous()
        return C.c_void_p(x.data_ptr())
    return C.c_void_p(int(x))


class Context:
    """One dgpu_ctx (one CUDA device, one host thread)."""

    def __init__(self, device=0):
        self._lib = lib()
        h = C.c_void_p()
        rc = self._lib.dgpu_ctx_create(int(device), C.byref(h))
        if rc != 0:
            raise DgpuError(f"dgpu_ctx_create(device={device}) failed: {self._lib.dgpu_strerror(rc).decode()}")
        self.h = h
        self.device = device

    def close(self):
        if self.h:
            self._lib.dgpu_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc, what):
        if rc != 0:
            raise DgpuError(f"{what} failed: {self._lib.dgpu_strerror(rc).decode()} "
                            f"[{self._lib.dgpu_last_error(self.h).decode()}]")

    def sync(self):
        self.check(self._lib.dgpu_ctx_sync(self.h), "dgpu_ctx_sync")

    def set_profiling(self, on=True):
        self.check(self._lib.dgpu_set_profiling(self.h, 1 if on else 0), "dgpu_set_profiling")

    def last_kernel_ms(self):
        return float(self._lib.dgpu_last_kernel_ms(self.h))

    def int_peak_tops(self):
        t = C.c_double()
        self.check(self._lib.dgpu_int_peak(self.h, C.byref(t)), "dgpu_int_peak")
        return t.value

    def int_peak_mix(self):
        """1e12 instructions/s of LOP3 chains alone, with IMAD chains interleaved, and with IMAD.WIDE.U32 chains interleaved."""
        t = (C.c_double * 3)()
        self.check(self._lib.dgpu_int_peak_mix(self.h, t), "dgpu_int_peak_mix")
        return {"lop3": t[0], "lop3_imad": t[1], "lop3_imad_wide": t[2]}

    @property
    def launches(self):
        return int(self._lib.dgpu_launch_count(self.h))

    @property
    def unsupported(self):
        """dgpu_unsupported_count: jobs refused per item so far (reads the device counters of asynchronous longNeedle and edit-path calls)."""
        self._lib.dgpu_unsupported_count.restype = C.c_uint64
        return int(self._lib.dgpu_unsupported_count(self.h))

    def set_ln_async_bound(self, max_cons, max_ref):
        """dgpu_set_ln_async_bound: no later longNeedle job exceeds max_cons x max_ref, so long_needle_dev reads nothing back and can be
        captured into a CUDA graph; (0, 0) switches back."""
        self.check(self._lib.dgpu_set_ln_async_bound(self.h, C.c_uint32(int(max_cons)), C.c_uint32(int(max_ref))), "dgpu_set_ln_async_bound")

    def set_msa_async_bound(self, max_reads, max_read_len):
        """dgpu_set_msa_async_bound: reserves the MSA workspace for clusters of up to max_reads reads, so msa_dev never grows it; (0, 0)
        switches back."""
        self.check(self._lib.dgpu_set_msa_async_bound(self.h, C.c_uint32(int(max_reads)), C.c_uint32(int(max_read_len))),
                   "dgpu_set_msa_async_bound")

    def set_ep_async_bound(self, max_query, max_target):
        """dgpu_set_ep_async_bound: no later edit-path job exceeds max_query x max_target, so edit_path_dev plans its Hirschberg levels on
        the device, reads nothing back and can be captured into a CUDA graph; (0, 0) switches back."""
        self.check(self._lib.dgpu_set_ep_async_bound(self.h, C.c_uint32(int(max_query)), C.c_uint32(int(max_target))), "dgpu_set_ep_async_bound")

    # ------------------------------------------------------------------ edit distance
    def edit_distance(self, seqs, q_off, q_len, t_off, t_len, k, mode, want_end=False):
        """Host form (numpy or pinned torch CPU tensors in, numpy out)."""
        n = len(q_off)
        dist = np.empty(n, np.int32)
        end = np.empty(n, np.int32) if want_end else None
        rc = self._lib.dgpu_edit_distance(self.h, _ptr(seqs), C.c_uint64(_nbytes(seqs)), _ptr(q_off), _ptr(q_len),
                                          _ptr(t_off), _ptr(t_len), _ptr(k), int(mode), C.c_uint64(n), _ptr(dist),
                                          _ptr(end))
        self.check(rc, "dgpu_edit_distance")
        return (dist, end) if want_end else dist

    def edit_distance_dev(self, seqs, q_off, q_len, t_off, t_len, k, mode, dist, end_loc=None, stream=None):
        """Device form: all arguments are CUDA tensors (uint8 / int32 storage), results written in place."""
        n = q_off.numel()
        rc = self._lib.dgpu_edit_distance_dev(self.h, _ptr(seqs), C.c_uint64(seqs.numel()), _ptr(q_off), _ptr(q_len),
                                              _ptr(t_off), _ptr(t_len), _ptr(k), int(mode), C.c_uint64(n), _ptr(dist),
                                              _ptr(end_loc), C.c_void_p(stream or 0))
        self.check(rc, "dgpu_edit_distance_dev")


    # ------------------------------------------------------------------ edit path
    def edit_path(self, seqs, q_off, q_len, t_off, t_len, mode, eq=b"", max_slice=None):
        """Host form. eq = additional equality pairs as bytes (first,second,...). Returns (dist, start, end, ops list[bytes], status).
        max_slice=None: dgpu_edit_path_ex (aligned target slices up to 16384 columns); otherwise dgpu_edit_path_wide, which traces slices
        up to max_slice (at most EP_MAX_SLICE) columns. Jobs with a wider slice come back with status 2."""
        n = len(q_off)
        cap = q_len.astype(np.uint64) + t_len.astype(np.uint64)
        ops_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64) if n else np.zeros(0, np.uint64)
        ops_bytes = int(cap.sum())
        ops = np.zeros(max(ops_bytes, 1), np.uint8)
        dist = np.zeros(n, np.int32); st = np.zeros(n, np.int32); en = np.zeros(n, np.int32)
        ops_len = np.zeros(n, np.uint32); status = np.zeros(n, np.uint32)
        args = (self.h, _ptr(seqs), C.c_uint64(_nbytes(seqs)), _ptr(q_off), _ptr(q_len), _ptr(t_off), _ptr(t_len), int(mode),
                C.c_char_p(eq) if eq else None, C.c_uint32(len(eq) // 2 if eq else 0), C.c_uint64(n), _ptr(dist), _ptr(st), _ptr(en),
                _ptr(ops), _ptr(ops_off), C.c_uint64(ops_bytes), _ptr(ops_len), _ptr(status))
        if max_slice is None:
            self.check(self._lib.dgpu_edit_path_ex(*args), "dgpu_edit_path_ex")
        else:
            self.check(self._lib.dgpu_edit_path_wide(*args, C.c_uint32(int(max_slice))), "dgpu_edit_path_wide")
        return dist, st, en, [ops[int(o):int(o) + int(l)].tobytes() for o, l in zip(ops_off, ops_len)], status

    def edit_path_dev(self, seqs, q_off, q_len, t_off, t_len, mode, dist, start, end, ops, ops_off, ops_len, status, eq=b"", stream=None,
                      max_slice=None):
        """Device form: CUDA tensors in, results written in place (ops at ops_off, |q| + |t| bytes reserved per job); max_slice as in
        edit_path."""
        n = q_off.numel()
        args = (self.h, _ptr(seqs), C.c_uint64(seqs.numel()), _ptr(q_off), _ptr(q_len), _ptr(t_off), _ptr(t_len), int(mode),
                C.c_char_p(eq) if eq else None, C.c_uint32(len(eq) // 2 if eq else 0), C.c_uint64(n), _ptr(dist), _ptr(start), _ptr(end),
                _ptr(ops), _ptr(ops_off), _ptr(ops_len), _ptr(status))
        if max_slice is None:
            self.check(self._lib.dgpu_edit_path_ex_dev(*args, C.c_void_p(stream or 0)), "dgpu_edit_path_ex_dev")
        else:
            self.check(self._lib.dgpu_edit_path_wide_dev(*args, C.c_uint32(int(max_slice)), C.c_void_p(stream or 0)), "dgpu_edit_path_wide_dev")

    # ------------------------------------------------------------------ longNeedle
    def long_needle(self, seqs, c_off, c_len, r_off, r_len, want_info=False, max_ref=None):
        """Host form. Returns (ok[uint8], aln_len[uint32], rows) where rows[i] = (row0 bytes, row1 bytes).
        max_ref=None: dgpu_long_needle (windows up to 16377 columns); otherwise dgpu_long_needle_ex, which also aligns wider windows
        up to max_ref (at most LN_MAX_REF) columns. Jobs beyond the limits come back with ok = 0."""
        n = len(c_off)
        cap = (c_len.astype(np.uint64) + r_len.astype(np.uint64))
        aln_off = np.concatenate([[0], np.cumsum(2 * cap)[:-1]]).astype(np.uint64) if n else np.zeros(0, np.uint64)
        aln_bytes = int(2 * cap.sum())
        aln = np.zeros(max(aln_bytes, 1), np.uint8)
        aln_len = np.zeros(n, np.uint32)
        ok = np.zeros(n, np.uint8)
        info = np.zeros((n, 4), np.int32) if want_info else None
        args = (self.h, _ptr(seqs), C.c_uint64(_nbytes(seqs)), _ptr(c_off), _ptr(c_len), _ptr(r_off), _ptr(r_len), C.c_uint64(n), _ptr(aln),
                _ptr(aln_off), C.c_uint64(aln_bytes), _ptr(aln_len), _ptr(ok), _ptr(info))
        if max_ref is None:
            self.check(self._lib.dgpu_long_needle(*args), "dgpu_long_needle")
        else:
            self.check(self._lib.dgpu_long_needle_ex(*args, C.c_uint32(int(max_ref))), "dgpu_long_needle_ex")
        rows = []
        for i in range(n):
            o, L, c = int(aln_off[i]), int(aln_len[i]), int(cap[i])
            rows.append((aln[o:o + L].tobytes(), aln[o + c:o + c + L].tobytes()))
        return (ok, aln_len, rows, info) if want_info else (ok, aln_len, rows)

    def long_needle_dev(self, seqs, c_off, c_len, r_off, r_len, aln, aln_off, aln_len, ok, info=None, stream=None, max_ref=None):
        """Device form (max_ref as in long_needle)."""
        n = c_off.numel()
        args = (self.h, _ptr(seqs), C.c_uint64(seqs.numel()), _ptr(c_off), _ptr(c_len), _ptr(r_off), _ptr(r_len), C.c_uint64(n), _ptr(aln),
                _ptr(aln_off), _ptr(aln_len), _ptr(ok), _ptr(info))
        if max_ref is None:
            self.check(self._lib.dgpu_long_needle_dev(*args, C.c_void_p(stream or 0)), "dgpu_long_needle_dev")
        else:
            self.check(self._lib.dgpu_long_needle_ex_dev(*args, C.c_uint32(int(max_ref)), C.c_void_p(stream or 0)), "dgpu_long_needle_ex_dev")


    # ------------------------------------------------------------------ msa
    def msa(self, seqs, read_off, read_len, cluster_off, sc=(5, -4, -10, -1), min_clique=2, want_alignment=False,
            check=True, max_reads=32):
        """Host form. Returns (consensus list[bytes], n_rows, status[, alignments list[list[bytes]]]).
        Clusters of more than max_reads (at most MSA_LARGE_MAXR) reads get status 1."""
        ncl = len(cluster_off) - 1
        rl = read_len.astype(np.uint64)
        csum = np.concatenate([[0], np.cumsum(rl)])
        cap = csum[cluster_off[1:]] - csum[cluster_off[:-1]]
        cons_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
        cons_bytes = int(cap.sum())
        cons = np.zeros(max(cons_bytes, 1), np.uint8)
        cons_len = np.zeros(ncl, np.uint32); n_rows = np.zeros(ncl, np.uint32); status = np.zeros(ncl, np.uint32)
        aln = aln_off = aln_cols = None
        aln_bytes = 0
        if want_alignment:
            nr = (cluster_off[1:] - cluster_off[:-1]).astype(np.uint64)
            acap = nr * 1024
            aln_off = np.concatenate([[0], np.cumsum(acap)[:-1]]).astype(np.uint64)
            aln_bytes = int(acap.sum())
            aln = np.zeros(max(aln_bytes, 1), np.uint8)
            aln_cols = np.zeros(ncl, np.uint32)
        rc = self._lib.dgpu_msa_ex(self.h, _ptr(seqs), C.c_uint64(_nbytes(seqs)), _ptr(read_off), _ptr(read_len),
                                   C.c_uint32(len(read_off)), _ptr(cluster_off), C.c_uint32(ncl), int(sc[0]), int(sc[1]),
                                   int(sc[2]), int(sc[3]), int(min_clique), _ptr(cons), _ptr(cons_off), C.c_uint64(cons_bytes),
                                   _ptr(cons_len), _ptr(n_rows), _ptr(status), _ptr(aln), _ptr(aln_off), C.c_uint64(aln_bytes),
                                   _ptr(aln_cols), C.c_uint32(max_reads))
        self.check(rc, "dgpu_msa_ex")
        if check and status.any():
            raise DgpuError(f"dgpu_msa_ex: {int((status != 0).sum())} cluster(s) rejected, first status codes "
                            f"{status[status != 0][:5].tolist()} (1 >{max_reads} reads, 2 too long, 3 non-ACGTN byte)")
        out = [cons[int(o):int(o) + int(l)].tobytes() for o, l in zip(cons_off, cons_len)]
        if not want_alignment:
            return out, n_rows, status
        alns = []
        for i in range(ncl):
            L, R, o = int(aln_cols[i]), int(n_rows[i]), int(aln_off[i])
            alns.append([aln[o + r * L:o + (r + 1) * L].tobytes() for r in range(R)])
        return out, n_rows, status, alns

    def msa_dev(self, seqs, read_off, read_len, cluster_off, ncl, sc, min_clique, cons, cons_off, cons_len, n_rows, status,
                stream=None, max_reads=32, aln=None, aln_off=None, aln_cols=None):
        """Device form: CUDA tensors in, results written in place; aln / aln_off / aln_cols (optional) receive the root alignments."""
        rc = self._lib.dgpu_msa_ex_dev(self.h, _ptr(seqs), C.c_uint64(seqs.numel()), _ptr(read_off), _ptr(read_len),
                                       _ptr(cluster_off), C.c_uint32(ncl), int(sc[0]), int(sc[1]), int(sc[2]), int(sc[3]),
                                       int(min_clique), _ptr(cons), _ptr(cons_off), _ptr(cons_len), _ptr(n_rows), _ptr(status),
                                       _ptr(aln), _ptr(aln_off), _ptr(aln_cols), C.c_uint32(max_reads), C.c_void_p(stream or 0))
        self.check(rc, "dgpu_msa_ex_dev")


def _nbytes(x):
    if isinstance(x, np.ndarray):
        return x.nbytes
    return x.numel() * x.element_size()
