"""ed_small_kernel (one thread per job, |q| <= 128): the DP column stays in registers, and every query length of the class against
150 bp targets matches the oracle, with N / IUPAC / lower-case bytes where the word-wise Peq build and the exact slow path meet."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from delly_b200 import synth
from oracle import pyoracle as po

ALPHA = np.frombuffer(b"ACGT", np.uint8)
ODD = np.frombuffer(b"NRYacgtn-", np.uint8)


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


def test_ed_small_kernel_has_no_stack_frame():
    """Every ed_small_kernel instantiation (NW 1-4 x NW/SHW/HW x with/without end locations) keeps its column in registers:
    a stack frame here means Pv / Mv / the shifted deltas went to local memory, which doubles the instructions of a column."""
    import delly_b200
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(delly_b200.LIB_PATH):
        pytest.skip("libdelly_b200.so not built")
    out = subprocess.run([exe, "-res-usage", delly_b200.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"STACK:(\d+)", line)
        if m and name and "ed_small_kernel" in name:
            found[name] = int(m.group(1))
        name = None
    assert len(found) == 24, sorted(found)
    assert all(v == 0 for v in found.values()), {k: v for k, v in found.items() if v}


def _jobs(seed):
    """For every |q| in 1..128 against 150 bp targets: related and unrelated pairs, and pairs whose query and / or target carry a byte
    outside ACGT (N, IUPAC, lower case) at the first, a middle or the last byte of a 4-byte word, at the 32-row word edges and on the
    query's last row. Some odd bytes occur in both sequences, so the exact slow path finds matches too."""
    rng = np.random.default_rng(seed)
    seqs, ks = [], []
    for ql in range(1, 129):
        for kind in range(8):
            t = ALPHA[rng.integers(0, 4, size=150)]
            if kind == 0:
                q = ALPHA[rng.integers(0, 4, size=ql)]
            else:
                a = int(rng.integers(0, 150 - min(ql, 150) + 1))
                q = synth.sub_noise(rng, t[a:a + ql], 0.05)[:ql].copy()
                if len(q) < ql:
                    q = np.concatenate([q, ALPHA[rng.integers(0, 4, size=ql - len(q))]])
            t = t.copy()
            if kind >= 2:
                # rows: word-of-four first / middle / last bytes, the 32-row word edges, the last row
                cand = [p for p in (0, 1, 2, 3, 4, 6, 7, 30, 31, 32, 33, 63, 64, 95, 96, 127) if p < ql] + [ql - 1]
                npos = 1 if kind in (2, 3) else int(rng.integers(1, 5))
                pos = [ql - 1] if kind == 3 else list(rng.choice(cand, size=npos))
                sym = ODD[rng.integers(0, len(ODD), size=len(pos))]
                if kind != 4:
                    q[pos] = sym
                if kind >= 4:
                    # the target gets the same odd bytes (matches through the slow path) and others, in the 16-column body and the tail
                    tp = rng.integers(0, 150, size=len(pos) + 2)
                    tp[-1] = int(rng.integers(144, 150))
                    t[tp] = np.concatenate([sym, ODD[rng.integers(0, len(ODD), size=2)]])
            seqs += [q, t]
            ks.append(-1 if kind % 3 else int(rng.integers(0, ql + 1)))
    arena, off, ln = synth.pack(seqs)
    return dict(seqs=arena, q_off=off[0::2].copy(), q_len=ln[0::2].copy(), t_off=off[1::2].copy(), t_len=ln[1::2].copy(),
                k=np.array(ks, np.int32))


def test_jobs_cover_every_query_length_and_odd_bytes():
    b = _jobs(7)
    assert sorted(set(b["q_len"].tolist())) == list(range(1, 129)) and set(b["t_len"].tolist()) == {150}
    odd = np.isin(b["seqs"], ODD)
    assert odd.sum() > 1000
    last = b["seqs"][(b["q_off"] + b["q_len"] - 1).astype(np.int64)]
    assert np.isin(last, ODD).sum() >= 128


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("want_end", [True, False])
def test_ed_small_kernel_matches_oracle_every_query_length(ctx, mode, want_end):
    b = _jobs(100 + mode)
    d, e = po.edit_distance_batch(po.oracle(), b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["k"], mode,
                                  threads=8, want_end=True)
    if want_end:
        gd, ge = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["k"], mode, want_end=True)
    else:
        gd = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["k"], mode)
    bad = np.nonzero(gd != d)[0]
    assert len(bad) == 0, (mode, bad[:5], gd[bad[:5]], d[bad[:5]], b["q_len"][bad[:5]])
    if want_end:
        ok = d >= 0
        bad = np.nonzero((ge != e) & ok)[0]
        assert len(bad) == 0, (mode, bad[:5], ge[bad[:5]], e[bad[:5]], b["q_len"][bad[:5]])
        assert np.all(ge[~ok] == -1)
