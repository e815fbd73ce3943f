"""The conv / linear GEMM's epilogue operands: the residual tile, loaded through TMA into shared memory during the k-loop,
and the bias2 rows and LayerNorm statistics, which idle producer warps stage into shared memory.

Cases the conformance matrix (test_gemm_matrix_gpu.py, whose case builder, sentinels, NaN poison and float64 reference
these tests reuse) does not reach:
  * narrow outputs with every operand: n_cols 4 (the UNet's output conv), 16 and 96;
  * residual boxes cut short by the output extent along W, H and N (TMA zero-fills them; no stored row reads one);
  * bias2 rows that change inside a tile: a row per output row, and groups that straddle frames and tile boundaries;
    conv boxes narrower than the frame (TW < oW or TH < oH) cover output rows that are not consecutive, so one tile can
    span more bias2 rows than it has rows (then each tile row gets its own staged bias2 row);
  * all of them under split-K, where every k-slice loads the residual and only the last one uses it;
  * a residual that is the output itself (in-place `out += f(x)`), read by TMA before any output is stored.
"""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

from test_gemm_matrix_gpu import (DEVICES, SENTINEL, SPLIT_K, _id, _m_box, _run, case,  # noqa: E402,F401
                                  ksplit_cap)

from tooncrafter_b200 import ops  # noqa: E402

NARROW_CASES = [
    case("linear", (300,), 128, 4, 16, bias=True, bias2=7, res=True),
    case("conv3x3", (3, 7, 9), 64, 4, 16, bias=True, res=True),
    case("linear", (300,), 128, 16, 16, bias2=3, scale=0.5, res=True),
    case("linear", (300,), 128, 96, 96, bias=True, bias2=1, res=True),
    case("conv3x3", (4, 5, 8), 64, 96, 96, bias=True, bias2=30, res=True),
]

# (TW, TH, TN) boxes ragged along W, H and N respectively
RAGGED_CASES = [
    case("conv3x3", (2, 3, 70), 64, 160, 160, bias=True, bias2=100, res=True),
    case("conv3x3", (3, 11, 13), 64, 200, 208, bias=True, res=True, scale=0.5),
    case("conv3x3", (7, 5, 8), 64, 256, 256, bias=True, bias2=45, res=True),
    case("conv3x3", (7, 5, 8), 64, 128, 128, res=True, row_stats=True),
]

# bias2 on conv boxes with gaps between their rows: spans of 182 and 325 bias2 rows (one staged row per tile row) and of
# 76 and 113 (one staged row per bias2 row the tile spans)
BIAS2_SPAN_CASES = [
    case("conv3x3", (2, 3, 70), 64, 160, 160, bias=True, bias2=1, res=True),
    case("conv3x3", (2, 3, 70), 64, 256, 256, bias2=1),
    case("conv3x3", (3, 11, 13), 64, 208, 208, bias=True, bias2=1, scale=0.5),
    case("conv3x3", (2, 10, 16), 64, 96, 96, bias=True, bias2=3, res=True),
    case("conv3x3", (2, 10, 16), 64, 256, 256, bias2=2),
]

SPLIT_CASES = [case("linear", (130,), SPLIT_K, 2 * bn, bn, bias=True, bias2=rp, res=True, ksplit=k)
               for bn, rp, k in ((96, 1, 2), (160, 5, 3), (256, 33, 4))]


def _bias2_span(c):
    """bias2 rows the tile of the case's first output row spans (the host's bound, reached by that tile here)."""
    N, H, W = c["geo"]
    TW, TH, TN = _m_box(N, H, W)
    extent = ((TN - 1) * H + (TH - 1)) * W + (TW - 1)
    return -(-extent // c["bias2"]) + 1


def test_case_tables_are_what_they_claim():
    ragged = []
    for c in RAGGED_CASES:
        N, H, W = c["geo"]
        TW, TH, TN = _m_box(N, H, W)
        ragged.append({d for d, extent, box in (("N", N, TN), ("H", H, TH), ("W", W, TW)) if extent % box})
    assert "W" in ragged[0] and "H" in ragged[1] and "N" in ragged[2], ragged
    spans = [_bias2_span(c) for c in BIAS2_SPAN_CASES]
    assert spans == [182, 182, 325, 76, 113], spans


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", NARROW_CASES + RAGGED_CASES + BIAS2_SPAN_CASES, ids=_id)
def test_epilogue_operands(c, dev, ksplit_cap):
    _run(c, dev, ksplit_cap)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", SPLIT_CASES, ids=_id)
def test_epilogue_operands_split_k(c, dev, ksplit_cap):
    _run(c, dev, ksplit_cap)


@pytest.mark.gpu
@pytest.mark.parametrize("geo,n,bn", [((1, 1, 300), 160, 160), ((3, 7, 9), 96, 96), ((7, 5, 8), 256, 256)])
def test_residual_is_the_output(geo, n, bn):
    """out = x @ w.T + bias + out on a window of a wider buffer; rows and columns outside the window keep the sentinel."""
    dev = "cuda"
    g = torch.Generator().manual_seed(n + bn)
    N, H, W = geo
    M, C = N * H * W, 64
    x = (torch.randn(M, C, generator=g)).half()
    w = (torch.randn(n, C, generator=g) * C ** -0.5).half()
    b = torch.randn(n, generator=g).float()
    r = torch.randn(M, n, generator=g).half()
    ldc, off = n + 24, 16
    out = torch.full((M + 2, ldc), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)
    win = torch.as_strided(out, (M, n), (ldc, 1), off)
    win.copy_(r.to(dev))
    ops.conv_gemm(x.to(dev), (N, H, W, C), (H * W * C, W * C, C), w.to(dev), ops.TAPS_1x1, out, geo, n, ldc=ldc,
                  out_offset=off, bias=b.to(dev), res=out, ldr=ldc, res_offset=off, block_n=bn)
    ref = x.double() @ w.double().t() + b.double() + r.double()
    got = win.cpu().double()
    assert torch.allclose(got, ref, rtol=2e-3, atol=1e-3), (got - ref).abs().max()
    bits = out.view(torch.int16).cpu().reshape(-1)
    keep = torch.ones_like(bits, dtype=torch.bool)
    keep[(off + torch.arange(M)[:, None] * ldc + torch.arange(n)[None]).reshape(-1)] = False
    assert ((bits == SENTINEL) | ~keep).all(), "wrote outside the output window"


@pytest.mark.gpu
def test_operands_too_large_for_shared_memory_are_refused():
    """A 256-wide tile with a residual and a bias2 row per output row needs the fp32 staging tile (130 KiB), the
    residual (64 KiB) and 128 bias2 rows (64 KiB): more shared memory than an SM has.  It is refused before launch."""
    from tooncrafter_b200 import _lib
    dev = "cuda"
    R, K, n = 256, 64, 256
    x = torch.randn(R, K, device=dev).half()
    w = torch.randn(n, K, device=dev).half()
    out = torch.zeros(R, n, dtype=torch.float16, device=dev)
    n0 = ops.launch_count()
    with pytest.raises(_lib.TcError, match="shared memory"):
        ops.linear(x, w, out, rows=R, K=K, n_cols=n, block_n=256, bias2=torch.zeros(R, n, dtype=torch.float16,
                   device=dev), bias2_rows_per=1, res=torch.zeros(R, n, dtype=torch.float16, device=dev))
    assert ops.launch_count() == n0
