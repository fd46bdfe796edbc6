"""Resources of every list kernel instance in the built library, read with cuobjdump (no GPU needed).

The list kernels take their image records by value in the kernel parameters (csrc/grl_param_list.cuh) and read them
from there.  A reference or pointer into the records that the compiler cannot fold away makes every thread copy the whole
list (up to 4 KB) to local memory: behaviour-neutral, and a large slowdown.  So every instance must use no stack and no
local memory.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "grl-image-restoration_b200", "libgrl_b200.so")
ANON = "_GLOBAL__N__"  # the mangled name of an anonymous namespace starts with this

# (mangled-name fragment, instances): the kernel templates and the readers / scales they are instantiated for
KERNELS = {
    "mosaic_kernel": 1,
    "luma_kernel": 1,
    "awgn_kernel": 1,
    "gather_planes_kernel": 4,  # {fp32 planes, RGGB} x {whole images, tile windows}
    "gather_u8_kernel": 2,  # {whole images, tile windows}
    "crop_planes_kernel": 1,
    "crop_u8_kernel": 1,
    "tile_accumulate_kernel": 1,
    "tile_finish_f32_kernel": 1,
    "tile_finish_u8_kernel": 1,
    "jpeg_blocks_kernel": 1,
    "jpeg_rgb_kernel": 1,
    "imresize_kernel": 6,  # {fp32, uint8} x s = 2, 3, 4
}


def _instances():
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if tool is None:
        pytest.skip("cuobjdump is not available")
    if not os.path.exists(LIB):
        pytest.skip("libgrl_b200.so is not built")
    out = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = {}
    for m in re.finditer(r"Function (_ZN3grl\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out):
        name, reg, stack, local = m.group(1), *map(int, m.groups()[1:])
        kernel = next((k for k in KERNELS if re.search(rf"\d{k}[EI]", name) and ANON in name), None)
        if kernel is not None:
            found.setdefault(kernel, []).append((name, reg, stack, local))
    return found


def test_every_instance_is_present():
    assert {k: len(v) for k, v in _instances().items()} == KERNELS


def test_no_stack_and_no_local_memory():
    for kernel, rows in _instances().items():
        for name, _, stack, local in rows:
            assert stack == 0 and local == 0, (kernel, name, stack, local)
