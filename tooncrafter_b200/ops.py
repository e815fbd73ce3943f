"""Torch-tensor wrappers over the C ABI (include/tooncrafter_b200.h).

torch is plumbing only here: it owns device memory and the current stream; every op below is one (or a few)
launches of our own sm_90a kernels through ctypes.  There is no fallback path — a missing library raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import TC_EPI_GEGLU, TcAttention, TcConvGemm, check

GN_MAX_PARTIALS = 296
DDIM_PARTIALS = 64


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req_half(t: torch.Tensor, name: str) -> None:
    if t.dtype != torch.float16 or not t.is_cuda:
        raise TypeError(f"{name} must be a CUDA float16 tensor, got {t.dtype} on {t.device}")


# tap tables (dx, dy, dn) ------------------------------------------------------------------------------
TAPS_1x1 = [(0, 0, 0)]
TAPS_3x3 = [(dx, dy, 0) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]  # weight order [ky][kx]
TAPS_T3 = [(0, dt, 0) for dt in (-1, 0, 1)]  # temporal (3,1,1) conv on the [B][T][HW][C] view


def taps_3x3_stride2(n_frames: int, pad: int = 1):
    """3x3 / stride 2 conv over a phase-split input [4][N][H/2][W/2][C] (tc_phase_split2), `pad` zero rows / columns
    before the image: 1 for the UNet's pad-1 downsample, 0 for the VAE encoder's F.pad(x, (0, 1, 0, 1))
    (ae_modules.py:104-108).

    input row 2*y + ky - pad  ->  phase row parity (ky-pad) & 1, row offset (ky-pad) >> 1 (floor).
    """
    taps = []
    for ky in range(3):
        for kx in range(3):
            py, oy = (ky - pad) & 1, (ky - pad) >> 1
            px, ox = (kx - pad) & 1, (kx - pad) >> 1
            taps.append((ox, oy, (py * 2 + px) * n_frames))
    return taps


def conv_gemm(a: torch.Tensor, a_dims, a_strides, w: torch.Tensor, taps: Sequence, out: torch.Tensor,
              out_dims, n_cols: int, *, ldc: Optional[int] = None, bias: Optional[torch.Tensor] = None,
              bias2: Optional[torch.Tensor] = None, bias2_rows_per: int = 0, res: Optional[torch.Tensor] = None,
              ldr: Optional[int] = None, acc_scale: float = 1.0, geglu: bool = False, block_n: int = 0,
              a_offset: int = 0, out_offset: int = 0, res_offset: int = 0,
              ln_stats: Optional[torch.Tensor] = None, ln_u: Optional[torch.Tensor] = None,
              ln_nslots: int = 0, ln_eps: float = 1e-5, row_stats: Optional[torch.Tensor] = None,
              row_stats_slots: int = 0) -> None:
    """out = epilogue(im2col(a) @ w.T).  a_dims = (N, H, W, C), a_strides = (sN, sH, sW) in elements.

    `*_offset` are element offsets applied to the base pointers (channel-slice views).
    ln_nslots > 0: `ln_stats` holds [M][ln_nslots][2] partial row sums written by a producer launch (`row_stats=`,
    `row_stats_slots = ceil(n_cols / block_n)`) instead of finished {mean, rstd} pairs.
    """
    _req_half(a, "a"); _req_half(w, "w"); _req_half(out, "out")
    lib = _lib.load()
    d = TcConvGemm()
    d.a = a.data_ptr() + 2 * a_offset
    d.a_N, d.a_H, d.a_W, d.a_C = a_dims
    d.a_sN, d.a_sH, d.a_sW = a_strides
    d.b = w.data_ptr()
    d.b_rows = w.shape[0]
    d.ldb = w.stride(0)
    d.taps = len(taps)
    for i, (dx, dy, dn) in enumerate(taps):
        d.tap_dx[i], d.tap_dy[i], d.tap_dn[i] = dx, dy, dn
    d.oN, d.oH, d.oW = out_dims
    d.out = out.data_ptr() + 2 * out_offset
    d.ldc = ldc if ldc is not None else (n_cols // 2 if geglu else n_cols)
    d.n_cols = n_cols
    if bias is not None:
        if bias.dtype != torch.float32:
            raise TypeError("bias must be float32")
        d.bias = bias.data_ptr()
    if bias2 is not None:
        _req_half(bias2, "bias2")
        d.bias2 = bias2.data_ptr()
        d.bias2_ld = bias2.stride(0)
        d.bias2_rows_per = bias2_rows_per
    if res is not None:
        _req_half(res, "res")
        d.res = res.data_ptr() + 2 * res_offset
        d.ldr = ldr if ldr is not None else n_cols
    d.acc_scale = acc_scale
    d.flags = TC_EPI_GEGLU if geglu else 0
    d.block_n = block_n
    ws = _gemm_ws(out.device)
    d.workspace = ws.data_ptr()
    d.workspace_bytes = ws.numel()
    if ln_stats is not None:
        d.ln_stats = ln_stats.data_ptr()
        d.ln_u = ln_u.data_ptr()
        d.ln_nslots = ln_nslots
        d.ln_eps = ln_eps
    if row_stats is not None:
        if row_stats.dtype != torch.float32:
            raise TypeError("row_stats must be float32")
        d.row_stats = row_stats.data_ptr()
        d.row_stats_slots = row_stats_slots
    check(lib.tc_conv_gemm(C.byref(d), _stream()), "tc_conv_gemm")


def linear(x: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, rows: int, K: int, n_cols: int,
           ldx: Optional[int] = None, **kw) -> None:
    """out[rows][n] = x[rows][K] @ w[n][K].T (+ epilogue); x row stride ldx."""
    ldx = ldx if ldx is not None else K
    conv_gemm(x, (1, 1, rows, K), (rows * ldx, rows * ldx, ldx), w, TAPS_1x1, out, (1, 1, rows), n_cols, **kw)


_GEMM_WS = {}
GEMM_WS_BYTES = 96 << 20


def _gemm_ws(device) -> torch.Tensor:
    """Per-device split-K scratch of tc_conv_gemm (tickets at its head, zeroed once; launches on a stream are ordered)."""
    if device.type != "cuda":
        return torch.zeros(1, dtype=torch.uint8)
    ws = _GEMM_WS.get(device)
    if ws is None:
        ws = torch.zeros(GEMM_WS_BYTES, dtype=torch.uint8, device=device)
        _GEMM_WS[device] = ws
    return ws


def last_gemm_config() -> dict:
    """(tests / profiling) tile configuration of the most recent tc_conv_gemm launch."""
    out = (C.c_int * 4)()
    check(_lib.load().tc_debug_last_gemm_config(out), "tc_debug_last_gemm_config")
    return dict(block_n=out[0], pair=bool(out[1]), ksplit=out[2], stages=out[3])


_GN_WS = {}
_GN_WS_RETIRED = []


def _gn_ws(device, n_floats: int) -> torch.Tensor:
    """Per-device statistics scratch of tc_groupnorm, grown on demand.  A grown-out workspace is retired, never freed:
    CUDA graphs captured while it was current keep its address and still write to it when they are replayed."""
    ws = _GN_WS.get(device)
    if ws is None or ws.numel() < n_floats:
        if ws is not None:
            _GN_WS_RETIRED.append(ws)
        ws = torch.empty(max(n_floats, 1 << 20), dtype=torch.float32, device=device)
        _GN_WS[device] = ws
    return ws


def groupnorm(x: torch.Tensor, y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *, frames: int,
              frames_per_stat: int, hw: int, C: int, G: int = 32, eps: float = 1e-5, silu: bool = False,
              ldx: Optional[int] = None, ldy: Optional[int] = None, x_offset: int = 0, y_offset: int = 0,
              ws: Optional[torch.Tensor] = None) -> None:
    _req_half(x, "x"); _req_half(y, "y")
    lib = _lib.load()
    n_stat = frames // frames_per_stat
    if ws is None:
        ws = _gn_ws(x.device, 2 * n_stat * G * GN_MAX_PARTIALS)
    check(lib.tc_groupnorm(x.data_ptr() + 2 * x_offset, ldx if ldx is not None else C,
                           y.data_ptr() + 2 * y_offset, ldy if ldy is not None else C,
                           gamma.data_ptr(), beta.data_ptr(), frames, frames_per_stat, hw, C, G, eps,
                           1 if silu else 0, ws.data_ptr(), _stream()), "tc_groupnorm")


def row_stats(x: torch.Tensor, stats: torch.Tensor, *, rows: int, C: int, eps: float = 1e-5,
              ldx: Optional[int] = None) -> None:
    """stats[r] = (mean, rstd) of row r (LayerNorm statistics; the affine part is folded into the next GEMM)."""
    _req_half(x, "x")
    lib = _lib.load()
    check(lib.tc_row_stats(x.data_ptr(), ldx if ldx is not None else C, rows, C, eps, stats.data_ptr(), _stream()),
          "tc_row_stats")


def layernorm(x: torch.Tensor, y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *, rows: int, C: int,
              eps: float = 1e-5, ldx: Optional[int] = None, ldy: Optional[int] = None) -> None:
    _req_half(x, "x"); _req_half(y, "y")
    lib = _lib.load()
    check(lib.tc_layernorm(x.data_ptr(), ldx if ldx is not None else C, y.data_ptr(),
                           ldy if ldy is not None else C, gamma.data_ptr(), beta.data_ptr(), rows, C, eps,
                           _stream()), "tc_layernorm")


def attention(q: torch.Tensor, segs, out: torch.Tensor, *, q_batches: int, Lq: int, heads: int, scale: float,
              ldq: int, ldo: int, q_offset: int = 0, out_offset: int = 0, head_dim: int = 64,
              causal: bool = False) -> None:
    """segs: list of dicts {k, v, ldk, ldv, Lk, kv_div, k_offset, v_offset} (1 or 2 segments).

    head_dim 64 or 80; causal masks key j for query i when j > i.  Head dim 80 and causal take one segment."""
    _req_half(q, "q"); _req_half(out, "out")
    lib = _lib.load()
    d = TcAttention()
    d.q = q.data_ptr() + 2 * q_offset
    d.ldq = ldq
    d.q_batches, d.Lq, d.heads = q_batches, Lq, heads
    d.n_seg = len(segs)
    for i, s in enumerate(segs):
        d.k[i] = s["k"].data_ptr() + 2 * s.get("k_offset", 0)
        d.v[i] = s["v"].data_ptr() + 2 * s.get("v_offset", 0)
        d.ldk[i], d.ldv[i] = s["ldk"], s["ldv"]
        d.Lk[i], d.kv_div[i] = s["Lk"], s.get("kv_div", 1)
    d.out = out.data_ptr() + 2 * out_offset
    d.ldo = ldo
    d.scale = scale
    d.head_dim = head_dim
    d.causal = 1 if causal else 0
    check(lib.tc_attention(C.byref(d), _stream()), "tc_attention")


def temporal_attention(q, k, v, out, *, ld: int, ldo: int, B: int, T: int, P: int, heads: int, scale: float,
                       q_offset: int = 0, k_offset: int = 0, v_offset: int = 0) -> None:
    lib = _lib.load()
    check(lib.tc_temporal_attention(q.data_ptr() + 2 * q_offset, k.data_ptr() + 2 * k_offset,
                                    v.data_ptr() + 2 * v_offset, ld, out.data_ptr(), ldo, B, T, P, heads, scale,
                                    _stream()), "tc_temporal_attention")


def attention_wide(qkv: torch.Tensor, out: torch.Tensor, *, batches: int, L: int, D: int, scale: float, ld: int, ldo: int,
                   q_offset: int = 0, k_offset: int = 0, v_offset: int = 0, out_offset: int = 0) -> None:
    """Single-head attention with head dim D (<= 512) over [batches][L] tokens; q / k / v are channel slices (element
    offsets) of one tensor with row stride `ld` (VAE mid-block AttnBlock, autoencoder_dualref.py:172-206)."""
    _req_half(qkv, "qkv"); _req_half(out, "out")
    lib = _lib.load()
    base = qkv.data_ptr()
    check(lib.tc_attention_wide(base + 2 * q_offset, base + 2 * k_offset, base + 2 * v_offset, ld, ld, ld,
                                out.data_ptr() + 2 * out_offset, ldo, batches, L, L, D, scale, _stream()), "tc_attention_wide")


def softmax_rows(s: torch.Tensor, *, rows: int, cols: int, scale: float, lds: Optional[int] = None) -> None:
    lib = _lib.load()
    check(lib.tc_softmax_rows(s.data_ptr(), lds if lds is not None else cols, rows, cols, scale, _stream()),
          "tc_softmax_rows")


def ncthw_to_cl(x: torch.Tensor, y: torch.Tensor, *, B, C_, T, H, W, Cpad, coff=0, scale=1.0) -> None:
    if x.dtype != torch.float32 or not x.is_contiguous():
        raise TypeError("ncthw_to_cl: x must be contiguous float32")
    lib = _lib.load()
    check(lib.tc_ncthw_to_cl(x.data_ptr(), y.data_ptr(), B, C_, T, H, W, Cpad, coff, scale, _stream()),
          "tc_ncthw_to_cl")


def cl_to_ncthw(x: torch.Tensor, y: torch.Tensor, *, B, C_, T, H, W, ldx, x_offset=0) -> None:
    lib = _lib.load()
    check(lib.tc_cl_to_ncthw(x.data_ptr() + 2 * x_offset, ldx, y.data_ptr(), 1 if y.dtype == torch.float32 else 0, B, C_, T, H,
                             W, _stream()), "tc_cl_to_ncthw")


def upsample2x(x, y, *, N, H, W, C_) -> None:
    lib = _lib.load()
    check(lib.tc_upsample2x(x.data_ptr(), y.data_ptr(), N, H, W, C_, _stream()), "tc_upsample2x")


def phase_split2(x, y, *, N, H, W, C_) -> None:
    lib = _lib.load()
    check(lib.tc_phase_split2(x.data_ptr(), y.data_ptr(), N, H, W, C_, _stream()), "tc_phase_split2")


def copy2d(src, dst, *, rows, cols, lds, ldd, src_offset=0, dst_offset=0) -> None:
    lib = _lib.load()
    check(lib.tc_copy2d(src.data_ptr() + 2 * src_offset, lds, dst.data_ptr() + 2 * dst_offset, ldd, rows, cols,
                        _stream()), "tc_copy2d")


def add2d(x, y, *, rows, cols, ldx, ldy, x_offset=0, y_offset=0) -> None:
    lib = _lib.load()
    check(lib.tc_add2d(x.data_ptr() + 2 * x_offset, ldx, y.data_ptr() + 2 * y_offset, ldy, rows, cols,
                       _stream()), "tc_add2d")


def gelu2d(x, y, *, rows, cols, ldx, ldy, x_offset=0, y_offset=0) -> None:
    """y = GELU(x), exact erf form; y may alias x."""
    lib = _lib.load()
    check(lib.tc_gelu2d(x.data_ptr() + 2 * x_offset, ldx, y.data_ptr() + 2 * y_offset, ldy, rows, cols, _stream()),
          "tc_gelu2d")


def video_u8(x16: torch.Tensor, x14: Optional[torch.Tensor], out: torch.Tensor, *, f_begin: int, f_end: int,
             out_frame: int) -> None:
    """Frames [f_begin, f_end) of one segment -> out[out_frame + f - f_begin] (uint8 [F, H, W, 3]).

    x16: fp16 [T, 3, H, W] decoder output of the 16-frame pass; x14: None or the [T-2, 3, H, W] output of the
    14-frame pass, whose frames T/2-2, T/2-1 replace frames T/2-1, T/2.  u = uint8(((clamp(x, -1, 1) + 1) / 2) * 255)."""
    _req_half(x16, "x16")
    T, C3, H, W = x16.shape
    if C3 != 3 or not x16.is_contiguous():
        raise ValueError("video_u8: x16 must be a contiguous [T, 3, H, W] tensor")
    if x14 is not None:
        _req_half(x14, "x14")
        if tuple(x14.shape) != (T - 2, 3, H, W) or not x14.is_contiguous():
            raise ValueError(f"video_u8: x14 must be a contiguous [{T - 2}, 3, {H}, {W}] tensor")
    if out.dtype != torch.uint8 or not out.is_cuda or not out.is_contiguous() or tuple(out.shape[1:]) != (H, W, 3):
        raise ValueError(f"video_u8: out must be a contiguous CUDA uint8 [F, {H}, {W}, 3] tensor")
    if out_frame < 0 or out_frame + (f_end - f_begin) > out.shape[0]:
        raise ValueError("video_u8: the frame window does not fit the output")
    lib = _lib.load()
    check(lib.tc_video_u8(x16.data_ptr(), _ptr(x14), T, H, W, f_begin, f_end, out.data_ptr() + out_frame * H * W * 3,
                          _stream()), "tc_video_u8")


def time_embed(t: torch.Tensor, w1, b1, w2, b2, out: torch.Tensor, ws: torch.Tensor, *, dim: int, hidden: int,
               accumulate: bool) -> None:
    lib = _lib.load()
    check(lib.tc_time_embed(t.data_ptr(), t.shape[0], dim, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                            b2.data_ptr(), hidden, out.data_ptr(), 1 if accumulate else 0, ws.data_ptr(),
                            _stream()), "tc_time_embed")


def small_linear(x: torch.Tensor, w, bias, y: torch.Tensor, *, silu_in: bool) -> None:
    lib = _lib.load()
    B, K = x.shape
    J = w.shape[0]
    check(lib.tc_small_linear(x.data_ptr(), B, K, w.data_ptr(), _ptr(bias), J, y.data_ptr(), y.stride(0),
                              1 if silu_in else 0, _stream()), "tc_small_linear")


def ddim_step(e_c, e_uc, x, noise, x_prev, pred_x0, coef, ws, *, B: int, n: int) -> None:
    lib = _lib.load()
    check(lib.tc_ddim_step(e_c.data_ptr(), e_uc.data_ptr(), x.data_ptr(), noise.data_ptr(), x_prev.data_ptr(),
                           pred_x0.data_ptr(), coef.data_ptr(), B, n, ws.data_ptr(), _stream()), "tc_ddim_step")


def ddim_step3(e_c, e_uc, e_img, x, noise, x_prev, pred_x0, coef, ws, *, B: int, n: int) -> None:
    """Three-way guidance (text / image-without-text / unconditional) + the update; coef holds 9 floats."""
    lib = _lib.load()
    check(lib.tc_ddim_step3(e_c.data_ptr(), e_uc.data_ptr(), e_img.data_ptr(), x.data_ptr(), noise.data_ptr(),
                            x_prev.data_ptr(), pred_x0.data_ptr(), coef.data_ptr(), B, n, ws.data_ptr(), _stream()),
          "tc_ddim_step3")


def dpm_step(e_c, e_uc, x, noise, prev_pred_x0, x_prev, pred_x0, coef, ws, *, B: int, n: int) -> None:
    """ddim_step plus DPM-Solver++(2M)'s correction x_prev += coef[8] * (pred_x0 - prev_pred_x0); coef holds 9 floats.
    prev_pred_x0 (the previous step's pred_x0) must be a buffer other than pred_x0; coef[8] == 0 leaves it unread."""
    lib = _lib.load()
    check(lib.tc_dpm_step(e_c.data_ptr(), e_uc.data_ptr(), x.data_ptr(), noise.data_ptr(), prev_pred_x0.data_ptr(),
                          x_prev.data_ptr(), pred_x0.data_ptr(), coef.data_ptr(), B, n, ws.data_ptr(), _stream()),
          "tc_dpm_step")


def dpm_step3(e_c, e_uc, e_img, x, noise, prev_pred_x0, x_prev, pred_x0, coef, ws, *, B: int, n: int) -> None:
    """ddim_step3 plus the correction of dpm_step, whose weight is coef[9] (after cfg_img); coef holds 10 floats."""
    lib = _lib.load()
    check(lib.tc_dpm_step3(e_c.data_ptr(), e_uc.data_ptr(), e_img.data_ptr(), x.data_ptr(), noise.data_ptr(),
                           prev_pred_x0.data_ptr(), x_prev.data_ptr(), pred_x0.data_ptr(), coef.data_ptr(), B, n,
                           ws.data_ptr(), _stream()), "tc_dpm_step3")


def q_sample(x, x0, noise, mask, coef, *, B: int, n: int, clean: bool = False) -> None:
    """In place on x (fp32 [B][n]): q = x0 if clean else coef[2b]*x0 + coef[2b+1]*noise per row b, then x = q where
    mask is None, else q*mask + (1 - mask)*x.  torch's fp32 op order, bit for bit.  x0 / noise / mask: contiguous fp32
    [B][n] (noise may be None with clean); coef: device fp32 [2B] (may be None with clean)."""
    for name, t in (("x", x), ("x0", x0), ("noise", noise), ("mask", mask)):
        if t is None:
            continue
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or t.numel() != B * n:
            raise ValueError(f"q_sample: {name} must be a contiguous CUDA float32 tensor of {B} x {n} elements")
    if coef is not None and (coef.dtype != torch.float32 or not coef.is_cuda or coef.numel() < 2 * B):
        raise ValueError(f"q_sample: coef must be a CUDA float32 tensor of at least {2 * B} elements")
    lib = _lib.load()
    check(lib.tc_q_sample(x.data_ptr(), x0.data_ptr(), _ptr(noise), _ptr(mask), _ptr(coef), 1 if clean else 0, B, n,
                          _stream()), "tc_q_sample")


def launch_count() -> int:
    return int(_lib.load().tc_launch_count())
