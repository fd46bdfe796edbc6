"""Resources of every attn_tc_kernel instance in the built library, read with cuobjdump (no GPU needed).

Two CTAs of 288 threads (two consumer warpgroups and a producer warp) share an SM, so that the four consumer
warpgroups on it hide each other's MMA and load latency.  Registers are allocated per SM sub-partition: each of the four
holds 16,384 and serves a quarter of the resident warps, and a warp's registers come in units of 256 (8 per thread).
The 18 warps of two CTAs put 5 warps on some sub-partition, which leaves at most 16,384 / (5 x 32) = 102, so 96
registers per thread; at 104 only one CTA fits.  A spill would put the O accumulator in local memory around every key
tile.  The shared-memory side of the same bound is a static_assert on AttnSmem in attn_tc.cu.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "grl-image-restoration_b200", "libgrl_b200.so")
WARPS_PER_CTA = 288 // 32
CTAS_PER_SM = 2
SMSPS = 4
REGS_PER_SMSP = 16384


def _cuobjdump():
    return shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


def _instances():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump is not available")
    if not os.path.exists(LIB):
        pytest.skip("libgrl_b200.so is not built")
    out = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = {}
    for m in re.finditer(r"Function _ZN3grl2tc14attn_tc_kernelILi(\d+)ELi(\d+)ELi(\d)E\S*:\s*\n\s*REG:(\d+) STACK:(\d+)", out):
        kt, kw, var, reg, stack = map(int, m.groups())
        found[(kt, kw, var)] = (reg, stack)
    return found


def test_every_instance_is_present():
    # KW: the key-window widths with a vectorised bias path, 0 = generic; VAR: bf16 bit | ones-column bit
    expected = {(64, kw, var) for kw in (0, 8, 16, 32, 64, 128) for var in range(4)}
    assert set(_instances()) == expected


def _ctas_per_sm(reg):
    per_thread = (reg + 7) // 8 * 8  # allocation granularity: 256 registers per warp
    warps = SMSPS * (REGS_PER_SMSP // (per_thread * 32))  # resident warps the register file holds
    return warps // WARPS_PER_CTA


def test_register_model():
    assert _ctas_per_sm(96) == 2 and _ctas_per_sm(104) == 1 and _ctas_per_sm(112) == 1
    assert _ctas_per_sm(72) == 3 and _ctas_per_sm(80) == 2


def test_two_ctas_per_sm():
    for key, (reg, _) in _instances().items():
        assert _ctas_per_sm(reg) >= CTAS_PER_SM, (key, reg)


def test_no_spills():
    for key, (_, stack) in _instances().items():
        assert stack == 0, (key, stack)
