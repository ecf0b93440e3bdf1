"""From the built library's SASS (tools/sass_mix.py): ed_pair_kernel keeps both jobs' columns in registers, the Peq build of
ed_small_kernel gathers two bit planes per query word instead of five byte compares per symbol, and running two jobs per thread leaves
fewer integer-ALU instructions per job-column than ed_small_kernel's fast block."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import sass_mix  # noqa: E402

NW2_HW_PROLOGUE_ALU_MAX = 300     # job load + Peq build of ed_small_kernel<2, HW, false> (472 with five match4 per 4-byte group)
NW2_PAIR_ALU_PER_JOB_COLUMN_MAX = 19.5


@pytest.fixture(scope="module")
def lib():
    import delly_b200
    if sass_mix.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(delly_b200.LIB_PATH):
        pytest.skip("libdelly_b200.so not built")
    return delly_b200.LIB_PATH


def test_pair_kernels_have_no_stack_frame(lib):
    out = subprocess.run([sass_mix.cuobjdump(), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"STACK:(\d+)", line)
        if m and name and "ed_pair_kernel" in name:
            found[name] = int(m.group(1))
        name = None
    assert len(found) == 4, sorted(found)
    assert all(v == 0 for v in found.values()), found


def test_nw2_hw_prologue_alu(lib):
    pro = sass_mix.small_prologues(lib)
    assert pro["NW=2 HW"] <= NW2_HW_PROLOGUE_ALU_MAX, pro


def test_nw2_pair_alu_per_job_column(lib):
    pr = sass_mix.pair_report(lib)
    assert sorted(pr) == ["NW=1", "NW=2", "NW=3", "NW=4"], sorted(pr)
    assert pr["NW=2"]["lds"] == 2, pr["NW=2"]
    assert pr["NW=2"]["alu"] <= NW2_PAIR_ALU_PER_JOB_COLUMN_MAX, pr["NW=2"]
