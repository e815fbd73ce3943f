"""tc_temporal_attention for 16 < T <= 64 (temporal_attn_mma64_kernel, clips longer than the training length) with the
harness of test_attention_matrix_gpu.py: NaN in the operand memory outside the views, a sentinel around the output
window, a second launch bit-identical to the first, and no element outside rtol 1e-3 / atol 1e-4 of the float64
reference (P split into fp16 hi + lo parts).  Every T from 17 to 64 with ragged P and several head counts, one
grid-stride case per tile count, and T = 65 refused without a launch."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

from test_attention_matrix_gpu import (DEVICES, GPU_ONLY, _build_temporal, _check_outside, _run_twice, _tid,  # noqa: E402
                                       _launch_temporal, tcase)
from test_kernels_gpu import _close  # noqa: E402

from tooncrafter_b200 import ops  # noqa: E402

LONG_CASES = [tcase(1 + t % 3, t, 5 + 11 * t, 1 + t % 7) for t in range(17, 65)]          # every T, ragged P
# B * P * heads items over 16 CTAs of 4 warps per SM: several items per warp for each tile count (2, 3, 4 x 16 frames)
BIG_LONG = [tcase(2, 24, 1300, 10), tcase(2, 40, 1800, 5), tcase(2, 64, 1400, 10)]


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", LONG_CASES, ids=_tid)
def test_temporal_attention_long(c, dev):
    b = _build_temporal(c, dev)
    _run_twice(lambda: _launch_temporal(c, b, dev), b, dev)
    _check_outside(b["out"], b["window"], _tid(c))
    _close(b["window"].cpu(), b["ref"], _tid(c), ns_max=0.0)


@pytest.mark.parametrize("dev", GPU_ONLY)
@pytest.mark.parametrize("c", BIG_LONG, ids=_tid)
def test_temporal_attention_long_grid_stride(c, dev):
    warps = 16 * 4 * torch.cuda.get_device_properties(0).multi_processor_count
    assert c["B"] * c["P"] * c["heads"] >= 2 * warps
    test_temporal_attention_long(c, dev)


@pytest.mark.gpu
def test_temporal_attention_refuses_t65():
    from tooncrafter_b200 import _lib
    B, T, P, heads = 1, 65, 4, 1
    C = heads * 64
    qkv = torch.zeros(B * T * P, 3 * C, dtype=torch.float16, device="cuda")
    out = torch.zeros(B * T * P, C, dtype=torch.float16, device="cuda")
    n0 = ops.launch_count()
    with pytest.raises(_lib.TcError, match="T <= 64"):
        ops.temporal_attention(qkv, qkv, qkv, out, ld=3 * C, ldo=C, B=B, T=T, P=P, heads=heads, scale=0.125,
                               k_offset=C, v_offset=2 * C)
    assert ops.launch_count() == n0, "a refused launch still launched"
