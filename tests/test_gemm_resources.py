"""Resources of every gemm_tc_kernel instance in the built library, read with cuobjdump (no GPU needed).

Up to BN = 192 two CTAs of 256 threads share an SM, so that one tile's epilogue overlaps the other tile's loads and
MMAs: each quarter of an SM's register file (16,384 registers) serves 4 of the 16 warps, which leaves at most 128
registers per thread.  The shared-memory side of the same bound is a static_assert on GemmSmem in gemm_tc.cu.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "grl-image-restoration_b200", "libgrl_b200.so")
THREADS = 256
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
    for m in re.finditer(r"Function _ZN3grl2tc14gemm_tc_kernelILi(\d+)ELi(\d)ELb(\d)E\S*:\s*\n\s*REG:(\d+) STACK:(\d+)", out):
        bn, epi, conv, reg, stack = map(int, m.groups())
        found[(bn, epi, conv)] = (reg, stack)
    return found


def test_every_instance_is_present():
    found = _instances()
    expected = {(bn, epi, 0) for bn in (64, 128, 192, 256) for epi in (0, 1, 2)} | {(bn, 0, 1) for bn in (64, 128, 192, 256)}
    assert set(found) == expected


def test_two_ctas_per_sm_up_to_bn_192():
    for (bn, epi, conv), (reg, _) in _instances().items():
        if bn > 192:
            continue
        per_thread = (reg + 7) // 8 * 8  # allocation granularity
        warps_per_smsp = 2 * (THREADS // 32) // 4
        assert per_thread * 32 * warps_per_smsp <= REGS_PER_SMSP, (bn, epi, conv, reg)


def test_no_spills():
    for key, (_, stack) in _instances().items():
        assert stack == 0, (key, stack)
