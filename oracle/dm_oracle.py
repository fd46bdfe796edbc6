"""CPU restatement of the reference's MATLAB-style demosaic  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

dm_matlab (utils/utils_mosaic.py:36-111) is the dm task's input transform (engines/base.py:127-128): packed RGGB planes
(B, 4, h, w) -> RGB (B, 3, 2h, 2w).  Restated here in torch ops, in fp32 (the reference's own arithmetic: the same
conv2d of the same stacked filters) or float64, with the mutation controls of the demosaic tests and the rounding bound
their gates use.  oracle/make_golden_dm.py asserts that the fp32 restatement reproduces the unmodified reference bit for
bit and writes tests/golden/dm_*.npz.  Only tests/ and oracle/ import this file.
"""
import torch
import torch.nn.functional as F

# utils/utils_mosaic.py:44-84, before the 1/8 scale
DM_KERNELS = {
    "kgrb": [[0, 0, -1, 0, 0], [0, 0, 2, 0, 0], [-1, 2, 4, 2, -1], [0, 0, 2, 0, 0], [0, 0, -1, 0, 0]],
    "krbg0": [[0, 0, 0.5, 0, 0], [0, -1, 0, -1, 0], [-1, 4, 5, 4, -1], [0, -1, 0, -1, 0], [0, 0, 0.5, 0, 0]],
    "krbbr": [[0, 0, -1.5, 0, 0], [0, 2, 0, 2, 0], [-1.5, 0, 6, 0, -1.5], [0, 2, 0, 2, 0], [0, 0, -1.5, 0, 0]],
}
# (channel, row parity, column parity) -> response channel of the (kgrb, krbg0, krbg1, krbbr) stack; every other site keeps
# the raw mosaic value (utils_mosaic.py:92, :97-109)
DM_FILL = {(1, 0, 0): 0, (1, 1, 1): 0, (0, 0, 1): 1, (0, 1, 0): 2, (0, 1, 1): 3, (2, 0, 1): 2, (2, 1, 0): 1, (2, 0, 0): 3}
DM_MAX_TAPS = 11  # nonzero taps of krbg0 / krbg1 (kgrb and krbbr have 9)
DM_MUTATIONS = ("swap_krbg", "zero_pad", "grbg")


def dm_matlab(cfa4, dtype=torch.float32, mutation=None, absolute=False):
    """utils/utils_mosaic.py:36-111 in `dtype` torch ops: packed RGGB planes (B, 4, h, w) -> RGB (B, 3, 2h, 2w).
    mutation (test controls): "swap_krbg" exchanges krbg0 and krbg1, "zero_pad" pads the mosaic with zeros instead of
    reflecting it, "grbg" fills the channels as if the sensor's phase were GRBG (column parity flipped).  absolute=True
    returns sum_i |w_i| |m_i| of the response each output takes (0 at raw sites), the scale of its rounding error."""
    if mutation is not None and mutation not in DM_MUTATIONS:
        raise ValueError(f"unknown mutation {mutation!r}")
    x = cfa4.to(dtype)
    B, _, h, w = x.shape
    cfa = torch.zeros(B, 1, 2 * h, 2 * w, dtype=dtype)
    cfa[:, 0, 0::2, 0::2] = x[:, 0]
    cfa[:, 0, 0::2, 1::2] = x[:, 1]
    cfa[:, 0, 1::2, 0::2] = x[:, 2]
    cfa[:, 0, 1::2, 1::2] = x[:, 3]
    k = {n: torch.tensor(v, dtype=dtype) / 8 for n, v in DM_KERNELS.items()}
    k0, k1 = k["krbg0"], k["krbg0"].t()
    if mutation == "swap_krbg":
        k0, k1 = k1, k0
    stack = torch.stack((k["kgrb"], k0, k1, k["krbbr"])).unsqueeze(1)
    if absolute:
        cfa, stack = cfa.abs(), stack.abs()
    rgb = torch.zeros_like(cfa).repeat(1, 3, 1, 1) if absolute else cfa.repeat(1, 3, 1, 1)
    pad = F.pad(cfa, (2, 2, 2, 2), mode="constant" if mutation == "zero_pad" else "reflect")
    conv = F.conv2d(pad, stack)
    flip = 1 if mutation == "grbg" else 0
    for (c, py, px), f in DM_FILL.items():
        rgb[:, c, py::2, px ^ flip::2] = conv[:, f, py::2, px ^ flip::2]
    return rgb


def dm_matlab_bound(cfa4):
    """Per-output bound on |fp32 evaluation - exact| of dm_matlab for any summation order of a response's <= 11 products:
    gamma_11 * sum_i |w_i| |m_i| (the weights are exact; products and partial sums round once each), float64."""
    u = 2.0 ** -24
    n = DM_MAX_TAPS
    return dm_matlab(cfa4, torch.float64, absolute=True) * (n * u / (1 - n * u))
