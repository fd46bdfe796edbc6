"""Numerics contract of the tensor-core attention's softmax (csrc/attn_tc.cu), restated in torch on the CPU and checked against
an exact float64 softmax(x) V -- the arithmetic of Attention.attn after the affine transform (mixed_attn_block_efficient.py:77-94).

What the kernel does per query row, in the log2 domain (x = S + bias + mask, everything fp32 unless noted):
  * key tiles of 64; a running reference m_ref per row; P = exp2(x - m_ref) rounded to the 16-bit operand format;
  * O += P V on the tensor pipe (fp32 accumulate); the denominator is the fp32 sum of the ROUNDED P (the ones-column of V
    when head_dim < 32);
  * LAZY rescale (kTau = 8): the reference moves only when the maximum of a row of the warp (32 rows) outgrew its reference by
    more than 2^8 (always on the first tile); then every row of the warp takes delta = max(mx - m_ref, 0), scales O by 2^-delta.
The emulation (grl_oracle.lazy_softmax_emulate, also the reference of tests/test_gpu_tc_attn.py) is that algorithm, not
the kernel; it guards the design constants (kTau vs the fp16 range, 16-bit P with an fp32 denominator built from the same
rounded values) independently of any GPU."""
import pytest
import torch

from grl_oracle import ATTN_KEY_TILE as KT, ATTN_TAU as K_TAU, lazy_softmax_emulate

MASK_LOG2 = 100.0 * 1.4426950408889634  # the shift mask (-100) in the log2 domain


def emulate(x, v, fmt):
    """x (R, N) log2-domain scores, v (N, d) values (already in the operand format) -> (out (R, d), rescales per warp)."""
    out, info = lazy_softmax_emulate(x.double(), v.double(), torch.float16 if fmt == "fp16" else torch.bfloat16)
    assert info["p_max"] <= 2.0 ** K_TAU * (1 + 1e-6)  # the bound that keeps P inside the fp16 range
    return out, info["rescales"]


def exact(x, v):
    return torch.softmax(x.double() * 0.6931471805599453, dim=1) @ v.double()  # softmax of 2^x


def _case(name, R=128, N=1024, d=30):
    g = torch.Generator().manual_seed(1000 + CASES.index(name))
    v = torch.randn(N, d, generator=g).half().float()
    if name == "typical":  # cosine logits * scale (<= 100 log2e) + bias in (0, 16 log2e)
        x = torch.randn(R, N, generator=g) * 6 + torch.rand(R, N, generator=g) * 23
    elif name == "growing":  # the row maximum grows by > 2^8 on every tile: the rescale / recompute path every time
        x = torch.randn(R, N, generator=g) + (torch.arange(N) // KT * 9.0)[None, :]
    elif name == "shrinking":  # reference fixed by the first tile, later tiles far below it (P deep in the fp16 subnormals)
        x = torch.randn(R, N, generator=g) - (torch.arange(N) // KT * 3.0)[None, :]
    elif name == "masked":  # half of the keys carry the shift mask
        x = torch.randn(R, N, generator=g) * 4
        x[:, ::2] -= MASK_LOG2
    elif name == "first_tile_masked":  # the whole first tile is masked: the reference starts ~144 too low and must catch up
        x = torch.randn(R, N, generator=g) * 4
        x[:, :KT] -= MASK_LOG2
    elif name == "one_hot":  # a single dominant key per row, in a late tile
        x = torch.randn(R, N, generator=g)
        x[torch.arange(R), torch.randint(N // 2, N, (R,), generator=g)] += 60.0
    elif name == "constant":
        x = torch.full((R, N), 3.25)
    else:
        raise KeyError(name)
    return x, v


CASES = ["typical", "growing", "shrinking", "masked", "first_tile_masked", "one_hot", "constant"]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("fmt,tol", [("fp16", 1.5e-3), ("bf16", 1.2e-2)])
def test_lazy_rescale_softmax_matches_exact(name, fmt, tol):
    x, v = _case(name)
    got, rescales = emulate(x, v, fmt)
    want = exact(x, v)
    assert torch.isfinite(got).all()
    err = (got - want).abs().max().item() / max(want.abs().max().item(), 1e-6)
    assert err <= tol, (name, fmt, err)
    if name == "growing":
        assert rescales == (x.shape[0] // 32) * (x.shape[1] // KT - 1)  # every tile after the first, every warp
    if name in ("shrinking", "constant"):
        assert rescales == 0  # a reference that is already high enough never touches O again
    if name == "typical":
        assert rescales <= 0.4 * (x.shape[0] // 32) * (x.shape[1] // KT - 1)  # rare (the kernel measures ~7 % on cfg4)


def test_denominator_uses_the_rounded_probabilities():
    """Normalising by the fp32 sum of the ROUNDED P (what the ones-column of V yields) keeps the weights a partition of unity:
    a constant value vector comes back exactly (to fp32 rounding), which a denominator built from unrounded P would not."""
    x, _ = _case("typical", N=512)
    v = torch.full((512, 4), 0.75)
    got, _ = emulate(x, v, "fp16")
    assert (got - 0.75).abs().max().item() <= 2e-6
