"""ed_small_kernel's HW fast block (tools/sass_mix.py over the built library): the score is read at the fixed bit 31, so no column
shifts by a register amount, and the integer ALU pipe, which bounds the kernel, runs at most the instructions per column it reaches
with the cross-word shifts and the score update on the FMA pipe."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import sass_mix  # noqa: E402

# ALU instructions per column of the fast block of ed_small_kernel<NW, HW, false> (27 with the score read at bit |q| - 1)
NW2_HW_ALU_MAX = 21.5


@pytest.fixture(scope="module")
def mix():
    import delly_b200
    if sass_mix.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(delly_b200.LIB_PATH):
        pytest.skip("libdelly_b200.so not built")
    return sass_mix.report(delly_b200.LIB_PATH)


def test_hw_fast_blocks_have_no_variable_right_shift(mix):
    hw = {k: v for k, v in mix.items() if " HW" in k}
    assert len(hw) == 8, sorted(mix)
    assert all(v["lds"] == int(k[3]) for k, v in hw.items()), {k: v["lds"] for k, v in hw.items()}
    assert all(v["vshr"] == 0 for v in hw.values()), {k: v["vshr"] for k, v in hw.items()}


def test_nw2_hw_alu_per_column(mix):
    assert mix["NW=2 HW"]["alu"] <= NW2_HW_ALU_MAX, mix["NW=2 HW"]
