"""TEST INFRASTRUCTURE — a CPU interpreter for recorded engine programs.

The engines record flat lists of `tooncrafter_b200.ops.*` calls (tensor, geometry, offsets).  This module gives
every op a plain-PyTorch meaning (fp32 math, fp16 storage) so that the HOST logic — weight packing, buffer
slicing, strides, tap tables, program order, arena reuse — can be validated on a GPU-less machine against the
oracle.  It never runs in the product path and says nothing about the CUDA kernels (tests/test_kernels_gpu.py
does that on the H100).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _strided(t, size, stride, off=0):
    """as_strided relative to the tensor's own first element (arena tensors have a non-zero storage offset)."""
    return torch.as_strided(t, size, stride, t.storage_offset() + off)


def _view2d(t, rows, cols, ld, off):
    return _strided(t, (rows, cols), (ld, 1), off)


def conv_gemm(a, a_dims, a_strides, w, taps, out, out_dims, n_cols, *, ldc=None, bias=None, bias2=None,
              bias2_rows_per=0, res=None, ldr=None, acc_scale=1.0, geglu=False, block_n=0, a_offset=0,
              out_offset=0, res_offset=0, ln_stats=None, ln_u=None, ln_nslots=0, ln_eps=1e-5, row_stats=None,
              row_stats_slots=0):
    aN, aH, aW, C = a_dims
    sN, sH, sW = a_strides
    A = _strided(a, (aN, aH, aW, C), (sN, sH, sW, 1), a_offset).float()
    oN, oH, oW = out_dims
    n = torch.arange(oN).view(-1, 1, 1)
    y = torch.arange(oH).view(1, -1, 1)
    x = torch.arange(oW).view(1, 1, -1)
    cols = []
    for dx, dy, dn in taps:
        nn_, yy, xx = n + dn, y + dy, x + dx
        ok = (nn_ >= 0) & (nn_ < aN) & (yy >= 0) & (yy < aH) & (xx >= 0) & (xx < aW)
        g = A[nn_.clamp(0, aN - 1), yy.clamp(0, aH - 1), xx.clamp(0, aW - 1)]          # [oN, oH, oW, C]
        cols.append(g * ok.unsqueeze(-1))
    M = oN * oH * oW
    X = torch.cat(cols, dim=-1).reshape(M, len(taps) * C)
    assert w.shape[1] == len(taps) * C, f"weight K {w.shape[1]} != taps*C {len(taps) * C}"
    assert n_cols <= w.shape[0]
    assert not geglu or acc_scale == 1.0, "GEGLU takes no acc_scale"
    acc = X @ w[:n_cols].float().t()
    if ln_stats is not None and ln_nslots > 0:
        # partial {sum, sumsq} slots written by a producer launch (any slot layout: only the totals matter)
        ps = ln_stats.view(-1)[:M * ln_nslots * 2].view(M, ln_nslots, 2).float().sum(1)
        mean = ps[:, 0:1] / C
        rstd = torch.rsqrt((ps[:, 1:2] / C - mean * mean).clamp_min(0) + ln_eps)
        acc = rstd * (acc - mean * ln_u[:n_cols].float())
    elif ln_stats is not None:
        st = ln_stats.view(-1, 2)[:M].float()
        acc = st[:, 1:2] * (acc - st[:, 0:1] * ln_u[:n_cols].float())
    if bias is not None:
        acc = acc + bias[:n_cols].float()
    if geglu:
        bn = block_n
        hb = bn // 2
        t = acc.reshape(M, n_cols // bn, 2, hb)
        val = (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(M, n_cols // 2)
        width = n_cols // 2
    else:
        if bias2 is not None:
            grp = torch.arange(M) // bias2_rows_per
            acc = acc + bias2.float()[grp][:, :n_cols]
        acc = acc * acc_scale
        if res is not None:
            acc = acc + _view2d(res, M, n_cols, ldr, res_offset).float()
        val, width = acc, n_cols
    ldc = ldc if ldc is not None else width
    _view2d(out, M, width, ldc, out_offset).copy_(val.half())
    if row_stats is not None:
        assert block_n > 0 and row_stats_slots == -(-n_cols // block_n) and not geglu
        # slot j / block_n: the fp16-rounded outputs of one N tile
        q = F.pad(val.half().float(), (0, row_stats_slots * block_n - n_cols)).view(M, row_stats_slots, block_n)
        rs = row_stats.view(-1)[:M * row_stats_slots * 2].view(M, row_stats_slots, 2)
        rs[:, :, 0] = q.sum(2)
        rs[:, :, 1] = (q * q).sum(2)


def groupnorm(x, y, gamma, beta, *, frames, frames_per_stat, hw, C, G=32, eps=1e-5, silu=False, ldx=None, ldy=None,
              x_offset=0, y_offset=0, ws=None):
    ldx = ldx if ldx is not None else C
    ldy = ldy if ldy is not None else C
    rows = frames * hw
    X = _view2d(x, rows, C, ldx, x_offset).float()
    ns = frames // frames_per_stat
    v = X.reshape(ns, frames_per_stat * hw, C).permute(0, 2, 1)
    o = F.group_norm(v, G, gamma.float(), beta.float(), eps)
    if silu:
        o = F.silu(o)
    _view2d(y, rows, C, ldy, y_offset).copy_(o.permute(0, 2, 1).reshape(rows, C).half())


def row_stats(x, stats, *, rows, C, eps=1e-5, ldx=None):
    X = _view2d(x, rows, C, ldx if ldx is not None else C, 0).float()
    mean = X.mean(1)
    var = X.var(1, unbiased=False)
    stats.view(-1, 2)[:rows] = torch.stack([mean, torch.rsqrt(var + eps)], 1)


def layernorm(x, y, gamma, beta, *, rows, C, eps=1e-5, ldx=None, ldy=None):
    X = _view2d(x, rows, C, ldx if ldx is not None else C, 0).float()
    _view2d(y, rows, C, ldy if ldy is not None else C, 0).copy_(F.layer_norm(X, (C,), gamma.float(), beta.float(), eps).half())


def _heads(t, heads):
    b, l, _ = t.shape
    return t.reshape(b, l, heads, 64).transpose(1, 2)


def attention(q, segs, out, *, q_batches, Lq, heads, scale, ldq, ldo, q_offset=0, out_offset=0):
    C = heads * 64
    Q = _strided(q, (q_batches, Lq, C), (Lq * ldq, ldq, 1), q_offset).float()
    total = torch.zeros(q_batches, Lq, C)
    for s in segs:
        Lk, div = s["Lk"], s.get("kv_div", 1)
        kvb = (q_batches + div - 1) // div
        K = _strided(s["k"], (kvb, Lk, C), (Lk * s["ldk"], s["ldk"], 1), s.get("k_offset", 0)).float()
        V = _strided(s["v"], (kvb, Lk, C), (Lk * s["ldv"], s["ldv"], 1), s.get("v_offset", 0)).float()
        idx = torch.arange(q_batches) // div
        att = ((_heads(Q, heads) @ _heads(K[idx], heads).transpose(-1, -2)) * scale).softmax(-1) @ _heads(V[idx], heads)
        total += att.transpose(1, 2).reshape(q_batches, Lq, C)
    _strided(out, (q_batches, Lq, C), (Lq * ldo, ldo, 1), out_offset).copy_(total.half())


def temporal_attention(q, k, v, out, *, ld, ldo, B, T, P, heads, scale, q_offset=0, k_offset=0, v_offset=0):
    C = heads * 64

    def get(t, off):
        return _strided(t, (B, T, P, C), (T * P * ld, P * ld, ld, 1), off).float().permute(0, 2, 1, 3).reshape(B * P, T, C)

    Q, K, V = get(q, q_offset), get(k, k_offset), get(v, v_offset)
    att = ((_heads(Q, heads) @ _heads(K, heads).transpose(-1, -2)) * scale).softmax(-1) @ _heads(V, heads)
    o = att.transpose(1, 2).reshape(B, P, T, C).permute(0, 2, 1, 3)
    _strided(out, (B, T, P, C), (T * P * ldo, P * ldo, ldo, 1), 0).copy_(o.half())


def attention_wide(qkv, out, *, batches, L, D, scale, ld, ldo, q_offset=0, k_offset=0, v_offset=0, out_offset=0):
    get = lambda off: _strided(qkv, (batches, L, D), (L * ld, ld, 1), off).float()
    Q, K, V = get(q_offset), get(k_offset), get(v_offset)
    att = ((Q @ K.transpose(-1, -2)) * scale).softmax(-1) @ V
    _strided(out, (batches, L, D), (L * ldo, ldo, 1), out_offset).copy_(att.half())


def softmax_rows(s, *, rows, cols, scale, lds=None):
    v = _view2d(s, rows, cols, lds if lds is not None else cols, 0)
    v.copy_((v.float() * scale).softmax(-1).half())


def ncthw_to_cl(x, y, *, B, C_, T, H, W, Cpad, coff=0, scale=1.0):
    Y = y.view(B, T, H, W, Cpad)
    Y[..., coff:coff + C_] = (x.reshape(B, C_, T, H, W) * scale).permute(0, 2, 3, 4, 1).half()


def cl_to_ncthw(x, y, *, B, C_, T, H, W, ldx, x_offset=0):
    X = _strided(x, (B, T, H, W, C_), (T * H * W * ldx, H * W * ldx, W * ldx, ldx, 1), x_offset)
    y.view(B, C_, T, H, W).copy_(X.permute(0, 4, 1, 2, 3).to(y.dtype))


def upsample2x(x, y, *, N, H, W, C_):
    X = x[:N * H * W * C_].view(N, H, W, C_)
    y[:N * 4 * H * W * C_].view(N, 2 * H, 2 * W, C_).copy_(X.repeat_interleave(2, 1).repeat_interleave(2, 2))


def phase_split2(x, y, *, N, H, W, C_):
    X = x[:N * H * W * C_].view(N, H, W, C_)
    Y = y[:N * H * W * C_].view(4, N, H // 2, W // 2, C_)
    for ph in range(4):
        Y[ph] = X[:, (ph >> 1)::2, (ph & 1)::2]


def copy2d(src, dst, *, rows, cols, lds, ldd, src_offset=0, dst_offset=0):
    _view2d(dst, rows, cols, ldd, dst_offset).copy_(_view2d(src, rows, cols, lds, src_offset))


def add2d(x, y, *, rows, cols, ldx, ldy, x_offset=0, y_offset=0):
    v = _view2d(y, rows, cols, ldy, y_offset)
    v.copy_((v.float() + _view2d(x, rows, cols, ldx, x_offset).float()).half())


def gelu2d(x, y, *, rows, cols, ldx, ldy, x_offset=0, y_offset=0):
    _view2d(y, rows, cols, ldy, y_offset).copy_(F.gelu(_view2d(x, rows, cols, ldx, x_offset).float()).half())


def time_embed(t, w1, b1, w2, b2, out, ws, *, dim, hidden, accumulate):
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    a = t.float()[:, None] * freqs[None]
    e = torch.cat([a.cos(), a.sin()], -1)
    r = F.linear(F.silu(F.linear(e, w1.float(), b1)), w2.float(), b2)
    if accumulate:
        out += r
    else:
        out.copy_(r)


def small_linear(x, w, bias, y, *, silu_in):
    xi = F.silu(x.float()) if silu_in else x.float()
    y.copy_(F.linear(xi, w.float(), None if bias is None else bias.float()).to(y.dtype))


def ddim_step(e_c, e_uc, x, noise, x_prev, pred_x0, coef, ws, *, B, n, e_img=None):
    s, phi, sqrt_ac, sqrt_1mac, rescale, sqrt_aprev, dir_coef, sigma = [float(v) for v in coef[:8]]
    ec, eu = e_c.reshape(B, n), e_uc.reshape(B, n)
    if e_img is None:
        v = eu + s * (ec - eu)                           # half arithmetic, one rounding per op
    else:
        ei = e_img.reshape(B, n)
        v = eu + float(coef[8]) * (ei - eu) + s * (ec - ei)
    if phi > 0:
        ratio = ec.float().std(dim=1, keepdim=True).half() / v.float().std(dim=1, keepdim=True).half()
        v = phi * (v * ratio) + (1 - phi) * v
    v = v.float()
    xf, nz = x.reshape(B, n), noise.reshape(B, n)
    eps = sqrt_ac * v + sqrt_1mac * xf
    x0 = (sqrt_ac * xf - sqrt_1mac * v) * rescale
    pred_x0.reshape(B, n).copy_(x0)
    x_prev.reshape(B, n).copy_(sqrt_aprev * x0 + dir_coef * eps + sigma * nz)


def ddim_step3(e_c, e_uc, e_img, x, noise, x_prev, pred_x0, coef, ws, *, B, n):
    ddim_step(e_c, e_uc, x, noise, x_prev, pred_x0, coef, ws, B=B, n=n, e_img=e_img)


def video_u8(x16, x14, out, *, f_begin, f_end, out_frame):
    """Middle-frame splice (inference.py:270), frame window, then the save path of inference.py:148-153 in torch."""
    T = x16.shape[0]
    v = x16.clone()
    if x14 is not None:
        v[T // 2 - 1:T // 2 + 1] = x14[T // 2 - 2:T // 2]
    v = torch.clamp(v[f_begin:f_end].float(), -1.0, 1.0)
    v = (v + 1.0) / 2.0
    out[out_frame:out_frame + f_end - f_begin] = (v * 255).to(torch.uint8).permute(0, 2, 3, 1)


def q_sample(x, x0, noise, mask, coef, *, B, n, clean=False):
    """torch's fp32 arithmetic of ddpm3d.py:306-309 and ddim.py:172-180, in the reference's op order."""
    xv = x.reshape(B, n)
    x0v = x0.reshape(B, n)
    if clean:
        q = x0v.clone()
    else:
        c = coef[:2 * B].reshape(B, 2)
        q = c[:, :1] * x0v + c[:, 1:] * noise.reshape(B, n)
    if mask is not None:
        m = mask.reshape(B, n)
        q = q * m + (1.0 - m) * xv
    xv.copy_(q)


_TABLE = {f.__name__: f for f in (conv_gemm, groupnorm, row_stats, layernorm, attention, temporal_attention, softmax_rows, attention_wide,
                                  ncthw_to_cl, cl_to_ncthw, upsample2x, phase_split2, copy2d, add2d, time_embed,
                                  small_linear, ddim_step, ddim_step3, gelu2d, video_u8, q_sample)}


def executor(fn, args, kw):
    """Program.run(executor=...) hook: interpret one recorded ops.* call on CPU."""
    _TABLE[fn.__name__](*args, **kw)
