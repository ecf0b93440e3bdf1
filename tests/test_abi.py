"""The C-ABI shared library loads on a CPU-only box and exports every symbol include/dgpu.h declares.
No compute calls are made here (there is no GPU in the CPU test tier)."""
import ctypes as C
import os
import re

import pytest

import delly_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "dgpu.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(dgpu_[a-z0-9_]+)\s*\(", txt)))


def test_library_loads_and_exports_every_declared_symbol():
    lib = delly_b200.lib()
    syms = _declared_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(lib, s), f"{s} is declared in include/dgpu.h but not exported by libdelly_b200.so"


def test_version_and_error_strings():
    lib = delly_b200.lib()
    assert lib.dgpu_version() >= 1000
    assert b"no CPU fallback" in lib.dgpu_strerror(-3)


def test_context_creation_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    with pytest.raises(delly_b200.DgpuError):
        delly_b200.Context(0)


def test_host_mirror_library_loads():
    H = delly_b200.hostlib()
    for s in ("dh_cluster_sr", "dh_cluster_pe", "dh_select_junctions", "dh_align_consensus_batch", "dh_process_batch", "dh_msa_batch"):
        assert hasattr(H, s)


def test_product_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under delly_b200/ may reference it."""
    for dp, _, files in os.walk(os.path.join(ROOT, "delly_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".cpp", ".h")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                # comments may mention the checker; code must never import, load or link it
                assert "pyoracle" not in txt and "liboracle" not in txt and "libdelly_ref" not in txt, f
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f
                assert not re.search(r"#include\s+[<\"].*oracle", txt), f


@pytest.mark.gpu
def test_host_forms_check_caller_buffers(ctx):
    """ADVICE r1: a mis-sized caller buffer is an error code (DGPU_ERR_ARG = -2 / DGPU_ERR_CAPACITY = -4) before anything is launched"""
    import ctypes as C
    import numpy as np
    lib = ctx._lib
    arena = np.frombuffer(b"ACGTACGTACGTACGTACGTACGT" * 4, np.uint8).copy()
    p = lambda a: C.c_void_p(a.ctypes.data)
    qo = np.array([0], np.uint32); ql = np.array([40], np.uint32); to = np.array([40], np.uint32); tl = np.array([500], np.uint32)   # target runs off the arena
    dist = np.zeros(1, np.int32)
    assert lib.dgpu_edit_distance(ctx.h, p(arena), C.c_uint64(arena.nbytes), p(qo), p(ql), p(to), p(tl), None, 0, C.c_uint64(1), p(dist), None) == -2
    tl[0] = 40
    ops = np.zeros(16, np.uint8); oo = np.array([0], np.uint64); ol = np.zeros(1, np.uint32); st = np.zeros(1, np.uint32); s0 = np.zeros(1, np.int32); e0 = np.zeros(1, np.int32)
    rc = lib.dgpu_edit_path(ctx.h, p(arena), C.c_uint64(arena.nbytes), p(qo), p(ql), p(to), p(tl), 0, C.c_uint64(1), p(dist), p(s0), p(e0), p(ops), p(oo), C.c_uint64(16), p(ol), p(st))
    assert rc == -4                                     # the op slot needs |q| + |t| = 80 bytes, 16 were given
    aln = np.zeros(32, np.uint8); ao = np.array([0], np.uint64); al = np.zeros(1, np.uint32); ok = np.zeros(1, np.uint8)
    rc = lib.dgpu_long_needle(ctx.h, p(arena), C.c_uint64(arena.nbytes), p(qo), p(ql), p(to), p(tl), C.c_uint64(1), p(aln), p(ao), C.c_uint64(32), p(al), p(ok), None)
    assert rc == -4
    # dgpu_msa: two reads in one cluster; a consensus slot needs the cluster's total read length (80 bytes)
    ro = np.array([0, 40], np.uint32); rl = np.array([40, 40], np.uint32); cons = np.zeros(16, np.uint8); co = np.array([0], np.uint64)
    cl = np.zeros(1, np.uint32); nr = np.zeros(1, np.uint32); mst = np.zeros(1, np.uint32)
    msa = lambda coff, cons_bytes: lib.dgpu_msa(ctx.h, p(arena), C.c_uint64(arena.nbytes), p(ro), p(rl), C.c_uint32(2), p(coff), C.c_uint32(1),
                                                5, -4, -10, -1, 2, p(cons), p(co), C.c_uint64(cons_bytes), p(cl), p(nr), p(mst), None, None,
                                                C.c_uint64(0), None)
    rl[1] = 500
    assert msa(np.array([0, 2], np.uint32), 128) == -2      # the second read runs off the arena
    rl[1] = 40
    assert msa(np.array([0, 3], np.uint32), 128) == -2      # cluster_off is not a partition of the two reads
    assert msa(np.array([0, 2], np.uint32), 16) == -4       # the consensus slot needs 80 bytes, 16 were given
