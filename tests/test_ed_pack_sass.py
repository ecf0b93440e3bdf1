"""From the built library's SASS (tools/sass_mix.py): ed_pack_kernel keeps its packed column in registers, needs fewer integer-ALU
instructions per job-column than ed_pair_kernel for the probe lengths it takes over, and reads the score of the bottom query with a plain
IMAD and LEA.HI instead of a variable shift."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import sass_mix  # noqa: E402

PACK3_ALU_PER_JOB_COLUMN_MAX = 16.0        # ed_pair_kernel<2>: 19.1
PACK5_ALU_BELOW_NW3_PAIR = 3.0             # ed_pair_kernel<3>: 27.0


@pytest.fixture(scope="module")
def lib():
    import delly_b200
    if sass_mix.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(delly_b200.LIB_PATH):
        pytest.skip("libdelly_b200.so not built")
    return delly_b200.LIB_PATH


def test_pack_kernels_have_no_stack_frame(lib):
    out = subprocess.run([sass_mix.cuobjdump(), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+).*STACK:(\d+)", line)
        if m and name and "ed_pack_kernel" in name:
            found[name] = (int(m.group(1)), int(m.group(2)))
        name = None
    assert len(found) == 2, sorted(found)
    assert all(st == 0 for _, st in found.values()), found
    # 7 CTAs of 128 threads per SM for the 5-word column
    assert all(reg <= 72 for reg, _ in found.values()), found


def test_pack_alu_per_job_column(lib):
    pk, pr = sass_mix.pack_report(lib), sass_mix.pair_report(lib)
    assert sorted(pk) == ["W=3 WA=1", "W=5 WA=2"], sorted(pk)
    assert pk["W=3 WA=1"]["lds"] == 1.5 and pk["W=5 WA=2"]["lds"] == 2.5, pk
    assert pk["W=3 WA=1"]["alu"] <= PACK3_ALU_PER_JOB_COLUMN_MAX, pk["W=3 WA=1"]
    assert pk["W=5 WA=2"]["alu"] <= pr["NW=3"]["alu"] - PACK5_ALU_BELOW_NW3_PAIR, (pk["W=5 WA=2"], pr["NW=3"])
    assert all(v["vshr"] == 0 for v in pk.values()), pk


def test_bottom_score_read_is_imad_and_lea_hi(lib):
    """Per column: B's score = two LEA.HI of the top word, A's = an IMAD of word WA by the per-pair multiplier and two LEA.HI; no SHF.L
    by a register amount and no IMAD.HI / IMAD.WIDE beyond the shift carries (one IMAD.HI per Ph / Mh word)."""
    for name, lines in sass_mix.functions(sass_mix._sass(lib)).items():
        m = sass_mix.PACK_KERNEL.search(name)
        if not m:
            continue
        w = int(m.group(1))
        fast = max(sass_mix.blocks(lines), key=lambda b: sum(op.startswith("LDS") for op, _ in b))
        ops = [op for op, _ in fast]
        lea_hi = sum(op.startswith("LEA.HI") and "UR" not in a for op, a in fast)
        assert lea_hi == 4 * 4, (w, lea_hi)
        assert sum(op == "IMAD" and re.match(r"R\d+, R\d+(\.reuse)?, R\d+(\.reuse)?, RZ", a) is not None for op, a in fast) >= 2 * 4, w
        assert sum(op.startswith("IMAD.HI") for op in ops) <= 2 * w * 4, w
        assert not any(op.startswith("IMAD.WIDE") for op in ops), w
        assert not any(op.startswith("SHF.L") and re.match(r"\S+,\s*\S+,\s*R\d+(\.reuse)?,", a) for op, a in fast), w
