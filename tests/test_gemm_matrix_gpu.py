"""Conformance matrix of the conv / linear GEMM (tc_conv_gemm through ops.conv_gemm): every kernel instance
(kNJ = BNp / 32 = 1..8, BNp = block_n rounded up to 32), every legal block_n, split depths 2..4 with a short last slice,
and every epilogue, each against a float64 reference of the same operation on the same fp16-rounded inputs.

Every case also checks
  * the configuration that ran: ops.last_gemm_config() reports the forced block_n and the expected k-slices;
  * write bounds: the output is a window of a wider buffer (ldc > width, a non-zero out_offset, extra rows) prefilled with
    a sentinel bit pattern; everything outside [M, width] at the window must still hold it afterwards;
  * read bounds: operand memory outside the views is NaN (weight rows n_cols..b_rows and columns past K, A channels
    outside the slice and rows / frames past the grid, residual and bias2 columns past n_cols and rows past their last
    one, bias / ln_u entries past n_cols), so a padding row of the B box or a partial last tile that reaches a stored
    column shows up as a NaN in the result.

Tolerance: single-contraction epilogues are held to rtol 1e-3 / atol 1e-4 on every element (ns_max = 0: at most a
one-ulp fp16 rounding flip); folded-LayerNorm cases to the reference's own autocast arithmetic, as in
test_kernels_gpu.test_linear_with_folded_layernorm.

Each case runs twice: on the H100 (marked gpu) and on CPU through tests/ops_emulator.conv_gemm.  The CPU leg exercises
the case builders, sentinels, poison and float64 references without a GPU, and shows that the emulator the host-logic
tests rely on agrees with the reference on every epilogue combination.
"""
import re
import sys
import zlib
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

import ops_emulator  # noqa: E402
from test_kernels_gpu import _autocast_ln_linear, _close, _pack_conv_w, _viol_frac  # noqa: E402

from tooncrafter_b200 import engine, ops  # noqa: E402

DEVICES = [pytest.param("cpu", id="cpu"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]
WIDTHS = list(range(16, 257, 16))            # every legal block_n
WIDTHS32 = list(range(32, 257, 32))          # block_n without B-box padding rows (GEGLU, split-K)
SENTINEL = 0x5A5A                            # fp16 203.25: bit pattern of untouched output memory
_m = re.search(r"#define TC_GEMM_WS_TICKET_BYTES \((\d+) \* (\d+)\)",
               (HERE.parent / "include" / "tooncrafter_b200.h").read_text())
TICKET_BYTES = int(_m.group(1)) * int(_m.group(2))

_RAN = set()          # (BNp / 32, split) of every checked CUDA launch
_GEGLU_RAN = set()    # block_n of every checked CUDA GEGLU launch


def _r8(v):
    return (v + 7) // 8 * 8


def case(kind, geo, C, n, bn, **kw):
    """kind: linear (geo = (rows,)), conv3x3 / t3 (geo = (N, H, W) / (B, T, pixels)), stride2 (geo = output (N, H, W))."""
    c = dict(kind=kind, geo=tuple(geo), C=C, n=n, bn=bn, a_slice=False, bias=False, bias2=0, scale=1.0, res=False,
             geglu=False, ln=False, ksplit=1, row_stats=False)
    c.update(kw)
    return c


def _id(c):
    p = [c["kind"], "x".join(map(str, c["geo"])), f"C{c['C']}", f"n{c['n']}", f"bn{c['bn']}"]
    p += [k for k in ("a_slice", "bias", "res", "geglu", "ln", "row_stats") if c[k]]
    if c["bias2"]:
        p.append(f"bias2per{c['bias2']}")
    if c["scale"] != 1.0:
        p.append(f"scale{c['scale']}")
    if c["ksplit"] > 1:
        p.append(f"ks{c['ksplit']}")
    return "-".join(p)


def _m_box(oN, oH, oW):
    """The (TW, TH, TN) box of output pixels tc_conv_gemm tiles M with (same search as the host code)."""
    best, best_tiles = (1, 1, 1), -1
    for TW in range(1, min(oW, 128) + 1):
        for TH in range(1, min(128 // TW, oH) + 1):
            TN = min(128 // (TW * TH), oN)
            tiles = -(-oW // TW) * -(-oH // TH) * -(-oN // TN)
            if best_tiles < 0 or tiles < best_tiles or (tiles == best_tiles and (TW, TH) > best[:2]):
                best, best_tiles = (TW, TH, TN), tiles
    return best


# ------------------------------------------------------------------------------------------------ case builder
def _make(c, dev):
    """Operands (NaN outside their views), the output buffer (sentinel outside the window) and the float64 reference."""
    g = torch.Generator().manual_seed(zlib.crc32(_id(c).encode()))
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    kind, C, n, bn, geglu, ln = c["kind"], c["C"], c["n"], c["bn"], c["geglu"], c["ln"]
    a_ld, a_off = (C + 128, 64) if c["a_slice"] else (C, 0)
    nan16 = lambda *s: torch.full(s, float("nan"), dtype=torch.float16, device=dev)
    nan32 = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=dev)

    # A operand, laid out as the kernel reads it
    if kind == "linear":
        (R,) = c["geo"]
        M = R
        x16 = (rnd(R, C) * 3 + 0.7 if ln else rnd(R, C)).half()
        abuf = nan16(R + 2, a_ld)
        abuf[:R, a_off:a_off + C] = x16.to(dev)
        a_dims, a_strides, out_dims, taps = (1, 1, R, C), (R * a_ld, R * a_ld, a_ld), (1, 1, R), ops.TAPS_1x1
    else:
        N, H, W = c["geo"]
        M = N * H * W
        if kind == "stride2":
            x16 = rnd(N, 2 * H, 2 * W, C).half()
            # tc_phase_split2 layout [4][N][H][W][C], phase = row parity * 2 + column parity
            xa, NA = torch.cat([x16[:, py::2, px::2] for py in (0, 1) for px in (0, 1)]), 4 * N
            taps = ops.taps_3x3_stride2(N)
        else:
            x16 = xa = rnd(N, H, W, C).half()
            NA = N
            taps = ops.TAPS_3x3 if kind == "conv3x3" else ops.TAPS_T3
        abuf = nan16(NA + 1, H, W, a_ld)
        abuf[:NA, ..., a_off:a_off + C] = xa.to(dev)
        a_dims, a_strides, out_dims = (NA, H, W, C), (H * W * a_ld, W * a_ld, a_ld), (N, H, W)
    K = len(taps) * C
    x64 = x16.double()

    # weights in reference column order; GEGLU packs each N tile as [value (bn/2) | gate (bn/2)] (test_linear_geglu)
    inner, hb = n // 2, bn // 2
    perm = (torch.cat([torch.cat([torch.arange(i, i + hb), torch.arange(inner + i, inner + i + hb)])
                       for i in range(0, inner, hb)]) if geglu else torch.arange(n))
    bias_k = u_k = stats = ln_mod = w32 = b32 = None
    if ln:
        assert kind == "linear"
        ln_mod = torch.nn.LayerNorm(C)
        with torch.no_grad():
            ln_mod.weight.copy_(rnd(C) * 0.2 + 1.0)
            ln_mod.bias.copy_(rnd(C) * 0.2)
        w32, b32 = (rnd(n, C) * C ** -0.5).float(), rnd(n).float()
        f = engine.fold_layernorm(w32, b32, ln_mod, torch.device("cpu"), perm=perm if geglu else None)
        wk, bias_k, u_k = f.w, f.c, f.u
        xn = F.layer_norm(x64, (C,), ln_mod.weight.detach().double(), ln_mod.bias.detach().double(), 1e-5)
        h = xn @ w32.double().t() + b32.double()
        mean, var = x64.mean(1), x64.var(1, unbiased=False)
        stats = torch.stack([mean, (var + 1e-5).rsqrt()], 1).float()
    else:
        if kind == "linear":
            w16 = (rnd(n, K) * K ** -0.5).half()
            wk, h = w16[perm], x64 @ w16.double().t()
        elif kind in ("conv3x3", "stride2"):
            w16 = (rnd(n, C, 3, 3) * K ** -0.5).half()
            wk = _pack_conv_w(w16)
            h = F.conv2d(x64.permute(0, 3, 1, 2), w16.double(), padding=1, stride=2 if kind == "stride2" else 1)
            h = h.permute(0, 2, 3, 1).reshape(M, n)
        else:   # (3, 1, 1) Conv3d over T on the [B][T][pixels] view
            w16 = (rnd(n, C, 3) * K ** -0.5).half()
            wk = w16.permute(0, 2, 1).reshape(n, K)
            h = F.conv3d(x64.permute(0, 3, 1, 2)[..., None], w16.double()[..., None, None], padding=(1, 0, 0))
            h = h[..., 0].permute(0, 2, 3, 1).reshape(M, n)
        if c["bias"]:
            b = rnd(n)
            h, bias_k = h + b, b[perm].float()
    wbuf = nan16(n + 24, K + 64)            # b_rows > n_cols, ldb > K
    wbuf[:n, :K] = wk.to(dev)
    kw = dict(block_n=bn, geglu=geglu, a_offset=a_off)
    if bias_k is not None:
        kw["bias"] = nan32(n + 16)
        kw["bias"][:n] = bias_k.to(dev)
    if ln:
        kw["ln_u"] = nan32(n + 16)
        kw["ln_u"][:n] = u_k.to(dev)
        kw["ln_stats"] = nan32(M + 1, 2)
        kw["ln_stats"][:M] = stats.to(dev)

    if geglu:
        ref, width = h[:, :inner] * F.gelu(h[:, inner:]), inner
    else:
        if c["bias2"]:
            rp = c["bias2"]
            groups = -(-M // rp)
            b2 = (rnd(groups, n) * 0.5).half()
            kw["bias2"] = nan16(groups + 1, _r8(n) + 8)
            kw["bias2"][:groups, :n] = b2.to(dev)
            kw["bias2_rows_per"] = rp
            h = h + b2.double()[torch.arange(M) // rp]
        h = h * c["scale"]
        kw["acc_scale"] = c["scale"]
        if c["res"]:
            r16 = rnd(M, n).half()
            ldr = _r8(n) + 16
            kw["res"] = nan16(M + 1, ldr)
            kw["res"][:M, 8:8 + n] = r16.to(dev)
            kw.update(ldr=ldr, res_offset=8)
            h = h + r16.double()
        ref, width = h, n
    ldc = _r8(width) + 24
    out = torch.full((M + 2, ldc), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)
    kw.update(ldc=ldc, out_offset=16)
    if c["row_stats"]:
        kw["row_stats_slots"] = -(-n // bn)
        kw["row_stats"] = nan32(M + 1, kw["row_stats_slots"], 2)
    args = (abuf, a_dims, a_strides, wbuf[:, :K], taps, out, out_dims, n)
    return dict(args=args, kw=kw, ref=ref, out=out, M=M, width=width, ldc=ldc, x16=x16, ln=ln_mod, w32=w32, b32=b32,
                geglu=geglu)


def _launch(dev, args, kw, ksplit):
    if dev == "cpu":
        ops_emulator.conv_gemm(*args, **kw)
        return None
    ops.conv_gemm(*args, **kw)
    cfg = ops.last_gemm_config()
    bn = kw["block_n"]
    assert cfg["block_n"] == bn and cfg["ksplit"] == ksplit, f"ran {cfg}; expected block_n {bn}, {ksplit} k-slice(s)"
    _RAN.add(((bn + 31) // 32, ksplit > 1))
    if kw.get("geglu"):
        _GEGLU_RAN.add(bn)
    return cfg


def _window(b):
    return torch.as_strided(b["out"], (b["M"], b["width"]), (b["ldc"], 1), b["out"].storage_offset() + 16)


def _check_bounds(b, what):
    """Nothing outside the [M, width] window at out_offset changed."""
    M, width, ldc = b["M"], b["width"], b["ldc"]
    bits = b["out"].view(torch.int16).cpu().reshape(-1)
    keep = torch.ones_like(bits, dtype=torch.bool)
    keep[(16 + torch.arange(M)[:, None] * ldc + torch.arange(width)[None]).reshape(-1)] = False
    bad = ((bits != SENTINEL) & keep).nonzero()
    assert bad.numel() == 0, (f"{what}: wrote outside the output window, e.g. row {bad[0].item() // ldc} column "
                              f"{bad[0].item() % ldc - 16} of the window ({bad.numel()} elements)")


def _check(b, what, cfg):
    _check_bounds(b, what)
    out = _window(b).cpu()
    what = f"{what} {cfg or ''}"
    if b["ln"] is not None:
        # not a single contraction (fp16-rounded W * gamma, rstd * (acc - mean * u)): held to the reference's own
        # autocast arithmetic (fp16 LayerNorm output, fp16 weights) as the yardstick for the north-star fraction
        v16 = _viol_frac(_autocast_ln_linear(b["x16"], b["ln"], b["w32"], b["b32"], b.get("geglu", False), b["width"]), b["ref"])
        _close(out, b["ref"], f"{what} (autocast path: {100 * v16:.3f} % outside)", rel=4e-3, abs_=2e-3,
               ns_max=1.5 * v16 + 0.005)
    else:
        _close(out, b["ref"], what, ns_max=0.0)
    return out


def _run(c, dev, set_cap):
    set_cap(dev, c["ksplit"])
    b = _make(c, dev)
    cfg = _launch(dev, b["args"], b["kw"], c["ksplit"])
    _check(b, _id(c), cfg)
    return b, cfg


@pytest.fixture
def ksplit_cap():
    """set_cap(dev, cap): caps the k-slices of later CUDA launches (tc_debug_set_gemm_mode, process-global); the
    heuristic is restored after the test, also when it fails."""
    libs = []

    def set_cap(dev, cap):
        if dev != "cuda":
            return
        from tooncrafter_b200 import _lib
        lib = _lib.load()
        _lib.check(lib.tc_debug_set_gemm_mode(cap << 8), "tc_debug_set_gemm_mode")
        libs.append(lib)

    yield set_cap
    if libs:
        libs[0].tc_debug_set_gemm_mode(0)


# ------------------------------------------------------------------------------------------------ the matrix
# every block_n x (n_cols == block_n, a partial last N tile, n_cols % 8 != 0: scalar store / bias2 / residual path)
WIDTH_CASES = [case("linear", (129,), 128, n, bn, bias=True, bias2=50, res=True)
               for bn in WIDTHS for n in (bn, bn + (bn // 2) // 8 * 8, 2 * bn + 5)]

# one k-block; more k-blocks than pipeline stages (8 stages at block_n <= 32, 4 at 256: the ring phase wraps)
K_CASES = [case("linear", (200,), K, 2 * bn, bn, bias=True) for K in (64, 1088) for bn in (16, 96, 176, 256)]

ROW_CASES = [case("linear", (rows,), 192, 2 * bn + 8, bn, res=True) for rows in (1, 127, 128, 129, 300)
             for bn in (80, 224)]

GEOMETRY_CASES = [
    # 3x3 convs whose M box spans frames, with a ragged last box (9 taps: K = 9 C)
    case("conv3x3", (7, 5, 8), 128, 208, 112, bias=True, bias2=40),
    case("conv3x3", (3, 7, 9), 64, 100, 48, bias=True, res=True),
    case("conv3x3", (2, 10, 16), 64, 288, 144, bias=True, bias2=160),
    # stride 2 through the phase split, frame count not a multiple of the box's frames
    case("stride2", (4, 5, 8), 64, 128, 64, bias=True),
    case("stride2", (6, 4, 6), 128, 72, 16, bias=True, res=True),
    # temporal (3, 1, 1) conv over T with B > 1
    case("t3", (2, 5, 40), 128, 192, 96, bias=True, res=True, scale=0.5),
    case("t3", (3, 16, 10), 64, 200, 208, bias=True),
    # A is a channel slice of a wider tensor (a_sW > C, a_offset != 0)
    case("conv3x3", (2, 6, 10), 64, 240, 240, a_slice=True, bias=True),
    case("linear", (300,), 128, 160, 32, a_slice=True, res=True),
]

EPILOGUE_CASES = [
    case("linear", (300,), 128, 40, 16),                                    # none
    case("linear", (300,), 128, 424, 208),
    case("linear", (300,), 128, 136, 64, bias=True),                        # bias
    case("linear", (300,), 128, 357, 176, bias=True),
    case("conv3x3", (4, 5, 8), 64, 160, 80, bias=True, bias2=40),           # bias2 per frame (H W rows)
    case("conv3x3", (4, 5, 8), 64, 136, 128, bias=True, bias2=80),          # bias2 per sample (T H W rows, T = 2)
    case("linear", (300,), 128, 69, 32, bias=True, scale=0.5, res=True),    # acc_scale before the residual
    case("linear", (300,), 128, 480, 240, bias=True, bias2=100, scale=0.5, res=True),
    case("linear", (300,), 128, 117, 112, res=True),                        # residual: ldr != n_cols, res_offset
    case("linear", (300,), 128, 512, 256, res=True),
    case("linear", (300,), 128, 112, 48, ln=True),                          # folded LayerNorm, no GEGLU
    case("linear", (300,), 192, 432, 208, ln=True),
]

GEGLU_CASES = [case("linear", (160,), 128, 2 * bn, bn, geglu=True, bias=True, ln=ln) for bn in WIDTHS32
               for ln in (False, True)]

SPLIT_K = 64 * 179          # 179 k-blocks: the last of 2, 3 or 4 slices is one k-block short
SPLIT_CASES = [case("linear", (130,), SPLIT_K, 2 * bn, bn, bias=True, bias2=64, scale=0.5, res=True, ksplit=cap)
               for bn in WIDTHS32 for cap in (2, 3, 4)]
SPLIT_OTHER = case("linear", (300,), 64 * 40, 128, 64, bias=True)        # another split geometry between the runs


def _stats_n(bn):
    """Producer width: a multiple of 64 (it is the consumer's C), with a ragged last N tile where one exists."""
    cands = [n for n in range(64, 1025, 64) if n >= 2 * bn]
    return next((n for n in cands if n % bn), cands[0])


ROW_STATS_CASES = ([case("linear", (150,), 64, _stats_n(bn), bn, bias=True, res=True, row_stats=True) for bn in WIDTHS]
                   + [case("linear", (150,), 64, 1024, 16, bias=True, res=True, row_stats=True)]     # 64 slots
                   + [case("linear", (150,), 64, 2 * bn + 5, bn, bias=True, res=True, row_stats=True) for bn in WIDTHS])

REFUSED = ["bias2_misaligned", "bias2_ld", "geglu_acc_scale", "ldc_narrow", "ldr_narrow", "n_cols_past_b_rows"]


def test_case_tables_cover_what_they_claim():
    """Properties of the tables themselves (no launch): widths, tile raggedness, box geometry, split depths."""
    for c in WIDTH_CASES + K_CASES + ROW_CASES + GEOMETRY_CASES + EPILOGUE_CASES:
        assert not (c["ln"] and c["geglu"]) or c["n"] % c["bn"] == 0
    assert {c["bn"] for c in WIDTH_CASES} == set(WIDTHS)
    assert any(c["n"] % c["bn"] and c["n"] % 8 == 0 for c in WIDTH_CASES if c["bn"] % 32)
    assert {c["bn"] for c in GEGLU_CASES} == set(WIDTHS32)
    assert {(c["bn"], c["ksplit"]) for c in SPLIT_CASES} == {(bn, k) for bn in WIDTHS32 for k in (2, 3, 4)}
    for k in (2, 3, 4):
        per = -(-(SPLIT_K // 64) // k)
        assert SPLIT_K // 64 - (k - 1) * per < per, "every slice count leaves a short last slice"
    assert any(-(-n // 16) == 64 for n in (c["n"] for c in ROW_STATS_CASES if c["bn"] == 16))
    assert all(c["n"] % c["bn"] for c in ROW_STATS_CASES if c["bn"] not in (16, 32, 64))
    for c in GEOMETRY_CASES:
        if c["kind"] == "linear":
            continue
        N, H, W = c["geo"]
        TW, TH, TN = _m_box(N, H, W)
        if c["kind"] in ("conv3x3", "stride2") and not c["a_slice"]:
            assert TN > 1 and (N % TN or H % TH or W % TW), f"{_id(c)}: box {TW}x{TH}x{TN} is not ragged across frames"
        if c["kind"] == "stride2":
            assert N % TN, f"{_id(c)}: N is a multiple of the box's {TN} frames"


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", WIDTH_CASES, ids=_id)
def test_block_n_and_n_cols(c, dev, ksplit_cap):
    _run(c, dev, ksplit_cap)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", K_CASES, ids=_id)
def test_k_depth(c, dev, ksplit_cap):
    b, cfg = _run(c, dev, ksplit_cap)
    if cfg is not None and c["C"] > 64:
        assert cfg["stages"] < c["C"] // 64, f"{cfg}: the ring does not wrap"


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", ROW_CASES, ids=_id)
def test_linear_rows(c, dev, ksplit_cap):
    _run(c, dev, ksplit_cap)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", GEOMETRY_CASES, ids=_id)
def test_m_geometry(c, dev, ksplit_cap):
    _run(c, dev, ksplit_cap)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", EPILOGUE_CASES, ids=_id)
def test_epilogue(c, dev, ksplit_cap):
    _run(c, dev, ksplit_cap)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", GEGLU_CASES, ids=_id)
def test_geglu(c, dev, ksplit_cap):
    _run(c, dev, ksplit_cap)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", ROW_STATS_CASES, ids=_id)
def test_row_stats_producer_and_consumer(c, dev, ksplit_cap):
    """Producer: one {sum, sumsq} slot per N tile of the fp16 outputs, against float64 sums.  Consumer (producer width a
    multiple of 64): a LayerNorm-folded GEMM that reads the producer's output and its ln_nslots slots."""
    b, _ = _run(c, dev, ksplit_cap)
    M, n, bn = b["M"], c["n"], c["bn"]
    slots = b["kw"]["row_stats_slots"]
    rs = b["kw"]["row_stats"].cpu().double()
    q = F.pad(_window(b).cpu().double(), (0, slots * bn - n)).view(M, slots, bn)
    s1, s2, sabs = q.sum(2), (q * q).sum(2), q.abs().sum(2)
    tol = 256 * 2.0 ** -24              # worst case of an fp32 sum of at most 256 terms per slot
    assert ((rs[:M, :, 0] - s1).abs() <= tol * sabs + 1e-6).all(), f"{_id(c)}: slot sums"
    assert ((rs[:M, :, 1] - s2).abs() <= tol * s2 + 1e-6).all(), f"{_id(c)}: slot sums of squares"
    assert torch.isnan(rs[M]).all(), f"{_id(c)}: wrote statistics past the last row"
    if n % 64:
        return
    g = torch.Generator().manual_seed(n + bn)
    nc, bnc = 96, 48
    ln = torch.nn.LayerNorm(n)
    with torch.no_grad():
        ln.weight.copy_(torch.randn(n, generator=g) * 0.2 + 1.0)
        ln.bias.copy_(torch.randn(n, generator=g) * 0.2)
    w32, b32 = torch.randn(nc, n, generator=g) * n ** -0.5, torch.randn(nc, generator=g)
    f = engine.fold_layernorm(w32, b32, ln, torch.device("cpu"))
    wbuf = torch.full((nc + 8, n), float("nan"), dtype=torch.float16, device=dev)
    wbuf[:nc] = f.w.to(dev)
    u = torch.full((nc + 16,), float("nan"), device=dev)
    u[:nc] = f.u.to(dev)
    bias = torch.full((nc + 16,), float("nan"), device=dev)
    bias[:nc] = f.c.to(dev)
    ldc = nc + 8
    out = torch.full((M + 2, ldc), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)
    ld = b["ldc"]
    args = (b["out"], (1, 1, M, n), (M * ld, M * ld, ld), wbuf, ops.TAPS_1x1, out, (1, 1, M), nc)
    kw = dict(block_n=bnc, ldc=ldc, out_offset=16, a_offset=16, bias=bias, ln_stats=b["kw"]["row_stats"], ln_u=u,
              ln_nslots=slots, ln_eps=1e-5)
    cfg = _launch(dev, args, kw, 1)
    mid = _window(b).cpu()
    ref = F.layer_norm(mid.double(), (n,), ln.weight.detach().double(), ln.bias.detach().double(), 1e-5)
    ref = ref @ w32.double().t() + b32.double()
    bc = dict(out=out, M=M, width=nc, ldc=ldc, ref=ref, ln=ln, x16=mid, w32=w32, b32=b32, args=args)
    _check(bc, f"consumer of {slots} slots {_id(c)}", cfg)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", SPLIT_CASES, ids=_id)
def test_split_k(c, dev, ksplit_cap):
    """Split-K at every block_n that is a multiple of 32 and 2, 3 and 4 slices with a short last one: exactly the capped
    slice count runs, three runs are bitwise identical (slices summed in slice order), another split geometry launched
    in between finds the tickets zeroed and leaves them so, and the ticket words are zero afterwards."""
    ksplit_cap(dev, c["ksplit"])
    b = _make(c, dev)
    reps = 3 if dev == "cuda" else 1
    outs = []
    for rep in range(reps):
        b["out"].view(torch.int16).fill_(SENTINEL)
        cfg = _launch(dev, b["args"], b["kw"], c["ksplit"])
        outs.append(_window(b).clone())
        if rep == 0 and dev == "cuda":
            o = _make(SPLIT_OTHER, dev)
            _check(o, _id(SPLIT_OTHER), _launch(dev, o["args"], o["kw"], c["ksplit"]))
    for o in outs[1:]:
        assert torch.equal(outs[0], o), "split-K result differs run to run"
    _check(b, _id(c), cfg)
    if dev == "cuda":
        torch.cuda.synchronize()
        ws = ops._gemm_ws(b["out"].device)
        assert not ws[:TICKET_BYTES].any().item(), "split-K left a ticket word non-zero"


@pytest.mark.gpu
@pytest.mark.parametrize("form", REFUSED)
def test_refused_launch_arguments(form):
    """tc_conv_gemm refuses these forms before launching anything (include/tooncrafter_b200.h, TcConvGemm)."""
    from tooncrafter_b200 import _lib
    dev = "cuda"
    R, K, n = 64, 64, 16
    x = torch.randn(R, K, device=dev).half()
    w = torch.randn(n, K, device=dev).half()
    out = torch.zeros(R, n, dtype=torch.float16, device=dev)
    kw = dict(block_n=16, ldc=n)
    if form == "bias2_misaligned":          # 8 bytes past a 16-byte boundary
        kw["bias2"] = torch.zeros(2 * 24 + 8, dtype=torch.float16, device=dev)[4:4 + 2 * 24].view(2, 24)
        kw["bias2_rows_per"] = 32
    elif form == "bias2_ld":                # [B, 12]: rows 24 bytes apart
        n = 12
        kw["bias2"] = torch.zeros(2, 12, dtype=torch.float16, device=dev)
        kw["bias2_rows_per"] = 32
    elif form == "geglu_acc_scale":
        w = torch.randn(32, K, device=dev).half()
        n = 32
        kw.update(geglu=True, block_n=32, acc_scale=0.5)
    elif form == "ldc_narrow":
        kw["ldc"] = 8
    elif form == "ldr_narrow":
        kw["res"] = torch.zeros(R, 8, dtype=torch.float16, device=dev)
        kw["ldr"] = 8
    elif form == "n_cols_past_b_rows":
        w = w[:8]
    n0 = ops.launch_count()
    with pytest.raises(_lib.TcError, match="tc_conv_gemm"):
        ops.linear(x, w, out, rows=R, K=K, n_cols=n, **kw)
    assert ops.launch_count() == n0, "a refused launch still launched"
    print(f"{form}: {_lib.load().tc_last_error().decode()}")


_MATRIX = [WIDTH_CASES, K_CASES, ROW_CASES, GEOMETRY_CASES, EPILOGUE_CASES, GEGLU_CASES, ROW_STATS_CASES, SPLIT_CASES]


@pytest.mark.gpu
def test_matrix_ran_every_instance_unsplit_and_split(request):
    """Last in the file: the CUDA cases above ran kNJ = 1..8 both unsplit and split, and GEGLU at all eight widths."""
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node
            and getattr(it, "callspec", None) is not None and it.callspec.params.get("dev", "cuda") == "cuda"]
    expected = sum(len(t) for t in _MATRIX) + len(REFUSED)
    if len(mine) != expected:
        pytest.skip(f"{len(mine)} of the {expected} CUDA cases were selected")
    print("ran (kNJ, split):", sorted(_RAN), "GEGLU block_n:", sorted(_GEGLU_RAN))
    assert _RAN == {(k, s) for k in range(1, 9) for s in (False, True)}
    assert _GEGLU_RAN == set(WIDTHS32)
