"""Conformance matrix of the normalisation kernels: tc_groupnorm (gn_fused_kernel at every cluster size 1..8 the host
picks, and the two-kernel gn_stats_kernel + gn_apply_kernel path), tc_layernorm and tc_row_stats (kMaxVec 2, 5 and 8),
each against a float64 reference of the same operation on the same fp16-rounded inputs.

Every CUDA case also checks
  * the path that ran: a Python mirror of tc_groupnorm's host selection (_gn_plan) gives fused or two-pass, the
    cluster size, threads and blocks; the launch count moves by 1 (fused) or 2 (two-pass).  LayerNorm and row_stats
    pick kMaxVec from C;
  * write bounds: the output is a window of a wider buffer (row stride above C, a non-zero column offset, rows before and
    after) prefilled with a sentinel bit pattern that must be intact afterwards;
  * read bounds: input memory outside the view is NaN (channels outside the slice, rows past the last one);
  * determinism: a second launch gives a bitwise identical output, and in-place GroupNorm equals out-of-place.

Tolerance: rtol 1e-3 / atol 1e-4 on every element (ns_max = 0), as test_groupnorm, plus the max-norm bound of _close.
The inputs include a mean-offset sweep x = mu + sigma z with mu / sigma in {0, 4, 16, 64}, where statistics taken as
E[x^2] - E[x]^2 from fp32 sums would cancel, and groups of one constant value (output = beta).

Each case runs twice: on the H100 (marked gpu) and on CPU through tests/ops_emulator.py (cases above a few million
elements are CUDA-only).
"""
import sys
import zlib
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

import ops_emulator  # noqa: E402
from test_kernels_gpu import _close  # noqa: E402

from tooncrafter_b200 import ops  # noqa: E402

SENTINEL = 0x5A5A                            # fp16 203.25: bit pattern of untouched output memory
CPU_MAX_ELEMS = 3_000_000
PRODUCT_C = (128, 256, 320, 512, 640, 960, 1280, 1920, 2560)   # the GroupNorm widths the UNet and VAE run
PARTIAL_WARP_C = (96, 160, 192, 352, 576)                      # two-pass blocks that are not whole warps at G = 32
GN_MAX_PARTIALS = 296                                          # TC_GN_MAX_PARTIALS

_GN_RAN = set()       # ("fused", csize) / ("two",) of every checked CUDA GroupNorm launch
_LN_RAN = set()       # ("layernorm" | "row_stats", kMaxVec) of every checked CUDA launch


def _devices(n_elems):
    gpu = pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)
    return [pytest.param("cpu", id="cpu"), gpu] if n_elems <= CPU_MAX_ELEMS else [gpu]


def _seed(cid):
    return torch.Generator().manual_seed(zlib.crc32(cid.encode()))


def _sentinel(*s, dev):
    return torch.full(s, SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)


def _check_outside(buf, window, before, what):
    """Every element of `buf` outside `window` (a view into it) still holds its bits from `before` (a CPU copy)."""
    flat = buf.view(torch.int16).cpu().reshape(-1)
    keep = torch.ones_like(flat, dtype=torch.bool)
    idx = torch.as_strided(torch.arange(buf.numel()), window.shape, window.stride(),
                           window.storage_offset() - buf.storage_offset())
    keep[idx.reshape(-1)] = False
    bad = ((flat != before.view(torch.int16).reshape(-1)) & keep).nonzero()
    assert bad.numel() == 0, f"{what}: wrote outside the output window ({bad.numel()} elements, first at {bad[0].item()})"


def _offset_input(g, shape, mu):
    """fp16 x = mu + sigma z, sigma = 1 (mu / sigma = mu), as float64."""
    return (mu + torch.randn(*shape, generator=g, dtype=torch.float64)).half().double()


# ================================================================================================ GroupNorm
def _gn_plan(frames, fps, hw, C, G, sms):
    """Mirror of the launch selection in tc_groupnorm (csrc/tc_norm.cu): ("fused", csize, threads, blocks) or
    ("two", threads, nblk, nblk2)."""
    n_stat, pps, cpg = frames // fps, fps * hw, C // G
    if cpg % 8 == 0 and frames * hw * C * 2 <= (16 << 20):
        vpp = cpg // 8
        total_v = pps * vpp
        threads = (640 // (32 * vpp)) * (32 * vpp)
        if 32 % vpp == 0:
            threads = 640
        if threads >= 32 and total_v <= 8 * threads * 8:
            cs = 1
            while cs * threads * 8 < total_v + cs * (vpp + 1):
                cs += 1
            n_units = n_stat * G
            if cs <= 8 and (cs == 1 or n_units * cs <= 2 * sms):
                if cs == 1:
                    step = 32 if 32 % vpp == 0 else 32 * vpp
                    per_thread = 8 if n_units >= 4 * sms else 4
                    need = -(-total_v // per_thread)
                    threads = min(threads, max(step, -(-need // step) * step))
                return ("fused", cs, threads, n_units * cs)
    V = C // 8
    k = max(1, 512 // V)
    threads = -(-V * k // 32) * 32
    want = max(1, -(-pps // (4 * k)))
    cap = min(max(1, 2 * sms // n_stat), GN_MAX_PARTIALS)
    cap2 = max(1, 2 * sms // n_stat)
    return ("two", threads, min(want, cap), min(want, cap2))


def gcase(frames, fps, hw, C, G=32, silu=True, eps=1e-5, layout="slice", mu=0.0, const=False):
    return dict(frames=frames, fps=fps, hw=hw, C=C, G=G, silu=silu, eps=eps, layout=layout, mu=mu, const=const)


def _gid(c):
    p = [f"gn-{c['frames']}/{c['fps']}x{c['hw']}x{c['C']}", f"G{c['G']}", c["layout"], f"eps{c['eps']}"]
    p += ["silu"] if c["silu"] else []
    p += [f"mu{c['mu']:g}"] if c["mu"] else []
    p += ["const"] if c["const"] else []
    return "-".join(p)


GN_CASES = (
    # the product's widths, per-frame and per-clip statistics, ragged pixel counts, silu on and off, both epsilons
    [gcase(4, 1, 77, C, silu=i % 2 == 0, eps=1e-5 if i % 3 else 1e-6) for i, C in enumerate(PRODUCT_C)]
    + [gcase(8, 4, 7, C, silu=i % 2 == 1, layout="plain" if i % 2 else "slice") for i, C in enumerate(PRODUCT_C)]
    + [gcase(2, 2, 333, C, eps=1e-6) for C in (320, 1280, 2560)]
    # two-pass blocks that are not whole warps (G = 32, cpg 3..18), and G = 8 / 16 / 64 / 96
    + [gcase(3, 1, 333, C) for C in PARTIAL_WARP_C]
    + [gcase(4, 4, 7, C, silu=False) for C in PARTIAL_WARP_C]
    + [gcase(2, 1, 100, 96, G=8), gcase(2, 2, 50, 96, G=16), gcase(2, 1, 100, 192, G=64), gcase(2, 1, 50, 576, G=96),
       gcase(2, 1, 100, 352, G=16, eps=1e-6)]
    # C = 4096 (the largest width), hw = 1
    + [gcase(2, 1, 33, 4096), gcase(2, 2, 333, 4096, G=16), gcase(16, 16, 1, 512), gcase(6, 1, 1, 256),
       gcase(4, 2, 1, 96)]
    # every fused cluster size: 1..7 at G = 32 (the 16 MB cap), 8 at G = 16
    + [gcase(1, 1, hw, 1280) for hw in (1021, 1501, 2500, 3500, 4500, 5500, 6400)]
    + [gcase(1, 1, 3800, 1280, G=16), gcase(2, 2, 1000, 1280, G=8, silu=False)]
    # the two-kernel path for large tensors: per-clip and per-frame statistics, in place
    + [gcase(32, 16, 2560, 320), gcase(32, 1, 640, 640, layout="plain"), gcase(32, 16, 160, 1280, eps=1e-6)]
    # mean-offset sweep on the fused and the two-pass path
    + [gcase(1, 1, 1021, 1280, mu=mu) for mu in (4.0, 16.0, 64.0)]            # (mu = 0: the cluster-size case)
    + [gcase(2, 1, 3500, 1280, mu=mu) for mu in (4.0, 16.0, 64.0)]
    + [gcase(4, 1, 333, 960, mu=mu) for mu in (4.0, 16.0, 64.0)]
    + [gcase(3, 1, 333, 96, mu=mu) for mu in (4.0, 16.0, 64.0)]
    + [gcase(32, 16, 640, 320, mu=mu) for mu in (16.0, 64.0)]
    # a constant group (sigma = 0): output = beta, through SiLU when silu is on
    + [gcase(2, 1, 500, 640, const=True, silu=s) for s in (True, False)]
    + [gcase(4, 2, 300, 1280, const=True), gcase(3, 1, 333, 96, const=True, silu=False)]
)


def _build_gn(c, dev):
    g = _seed(_gid(c))
    frames, fps, hw, C, G = c["frames"], c["fps"], c["hw"], c["C"], c["G"]
    rows = frames * hw
    x64 = _offset_input(g, (rows, C), c["mu"])
    if c["const"]:
        x64[:, :C // G] = torch.tensor(2.7).half().double()         # norm group 0 of every stat group
    gamma = (torch.randn(C, generator=g, dtype=torch.float64) * 0.2 + 1.0).float()
    beta = (torch.randn(C, generator=g, dtype=torch.float64) * 0.2).float()
    if c["layout"] == "slice":
        ldx, xo, ldy, yo = C + 16, 8, C + 24, 16
    else:
        ldx, xo, ldy, yo = C, 0, C, 0
    xbuf = torch.full((rows + 1, ldx), float("nan"), dtype=torch.float16, device=dev)
    xbuf[:rows, xo:xo + C] = x64.half().to(dev)
    ybuf = _sentinel(rows + 2, ldy, dev=dev)
    kw = dict(frames=frames, frames_per_stat=fps, hw=hw, C=C, G=G, eps=c["eps"], silu=c["silu"], ldx=ldx, ldy=ldy,
              x_offset=xo, y_offset=ldy + yo)
    xr = x64.reshape(frames // fps, fps * hw, C).permute(0, 2, 1)
    ref = F.group_norm(xr, G, gamma.double(), beta.double(), c["eps"])
    if c["silu"]:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(rows, C)
    if c["const"]:
        b0 = beta.double()[:C // G]
        assert torch.allclose(ref[:, :C // G], F.silu(b0) if c["silu"] else b0.expand(rows, -1))
    return dict(xbuf=xbuf, ybuf=ybuf, kw=kw, ref=ref, gamma=gamma.to(dev), beta=beta.to(dev),
                window=ybuf[1:1 + rows, yo:yo + C], xwindow=xbuf[:rows, xo:xo + C])


def _gn(x, y, b, dev, **kw):
    if dev == "cpu":
        ops_emulator.groupnorm(x, y, b["gamma"], b["beta"], **kw)
    else:
        ops.groupnorm(x, y, b["gamma"], b["beta"], **kw)


@pytest.mark.parametrize("c,dev", [pytest.param(c, d.values[0], marks=d.marks, id=f"{_gid(c)}-{d.id}")
                                   for c in GN_CASES for d in _devices(c["frames"] * c["hw"] * c["C"])])
def test_groupnorm(c, dev):
    b = _build_gn(c, dev)
    kw = b["kw"]
    if dev == "cuda":
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        plan = _gn_plan(c["frames"], c["fps"], c["hw"], c["C"], c["G"], sms)
        n0 = ops.launch_count()
    _gn(b["xbuf"], b["ybuf"], b, dev, **kw)
    what = _gid(c)
    if dev == "cuda":
        assert ops.launch_count() - n0 == (1 if plan[0] == "fused" else 2), f"{what}: expected {plan}"
        what += f" {plan}"
        _GN_RAN.add(plan[:2] if plan[0] == "fused" else ("two",))
        first = b["window"].clone()
        b["window"].view(torch.int16).fill_(SENTINEL)
        _gn(b["xbuf"], b["ybuf"], b, dev, **kw)
        assert torch.equal(first.view(torch.int16), b["window"].view(torch.int16)), f"{what}: differs run to run"
        # in place, on the input's own slice
        z = b["xbuf"].clone()
        before = z.cpu()
        _gn(z, z, b, dev, **dict(kw, ldy=kw["ldx"], y_offset=kw["x_offset"]))
        zwin = z[:c["frames"] * c["hw"], kw["x_offset"]:kw["x_offset"] + c["C"]]
        assert torch.equal(zwin.view(torch.int16), first.view(torch.int16)), f"{what}: in place != out of place"
        _check_outside(z, zwin, before, what + " in place")
    _check_outside(b["ybuf"], b["window"], _sentinel(*b["ybuf"].shape, dev="cpu"), what)
    _close(b["window"].cpu(), b["ref"], what, ns_max=0.0)


def test_groupnorm_case_table_and_launch_shapes():
    """No launch: the table reaches every fused cluster size and the two-pass path on a 132-SM H100, and the two-pass
    block is a whole number of warps.  Rounding it up changes no launch of the product's widths."""
    plans = {_gn_plan(c["frames"], c["fps"], c["hw"], c["C"], c["G"], 132)[:2] for c in GN_CASES}
    assert {("fused", cs) for cs in range(1, 9)} <= plans and any(p[0] == "two" for p in plans)
    assert min(c["C"] // c["G"] for c in GN_CASES) == 3
    for C in PRODUCT_C + PARTIAL_WARP_C + (4096,):
        V = C // 8
        k = max(1, 512 // V)
        if C in PRODUCT_C:
            assert V * k % 32 == 0, f"C = {C}: the two-pass block of {V * k} threads would change"
        if C in PARTIAL_WARP_C:
            assert V * k % 32 != 0, f"C = {C}: {V * k} threads"
    for c in GN_CASES:
        p = _gn_plan(c["frames"], c["fps"], c["hw"], c["C"], c["G"], 132)
        if (c["C"] // c["G"]) % 8:
            assert p[0] == "two", _gid(c)


# ================================================================================================ LayerNorm / row_stats
LN_C = (8, 256, 512, 520, 1280, 1288, 2048)
LN_ROWS = (1, 7, 8, 9, 1000)


def lcase(rows, C, mu=0.0, strided=True, eps=1e-5):
    return dict(rows=rows, C=C, mu=mu, strided=strided, eps=eps)


def _lid(c):
    return f"{c['rows']}x{c['C']}" + ("-strided" if c["strided"] else "") + (f"-mu{c['mu']:g}" if c["mu"] else "") + (
        f"-eps{c['eps']}" if c["eps"] != 1e-5 else "")


def _kmaxvec(C):
    return 2 if C <= 512 else 5 if C <= 1280 else 8


LN_CASES = ([lcase(r, C, strided=(r + C) % 2 == 1 or r == 1000) for C in LN_C for r in LN_ROWS]
            + [lcase(300, C, mu=mu) for C in (256, 1280, 2048) for mu in (4.0, 16.0, 64.0)]
            + [lcase(77, 1024, eps=1e-6), lcase(9, 8, mu=64.0)])


def _build_ln(c, dev):
    g = _seed(_lid(c))
    rows, C = c["rows"], c["C"]
    x64 = _offset_input(g, (rows, C), c["mu"])
    gamma = (torch.randn(C, generator=g, dtype=torch.float64) * 0.2 + 1.0).float()
    beta = (torch.randn(C, generator=g, dtype=torch.float64) * 0.2).float()
    ldx, ldy = (C + 16, C + 24) if c["strided"] else (C, C)
    xbuf = torch.full((rows + 2, ldx), float("nan"), dtype=torch.float16, device=dev)
    x = xbuf[1:, 8:] if c["strided"] else xbuf[1:]
    x[:rows, :C] = x64.half().to(dev)
    ybuf = _sentinel(rows + 2, ldy, dev=dev)
    y = ybuf[1:, 16:] if c["strided"] else ybuf[1:]
    return dict(x=x, ldx=ldx, ybuf=ybuf, y=y, ldy=ldy, x64=x64, gamma=gamma.to(dev), beta=beta.to(dev),
                ref=F.layer_norm(x64, (C,), gamma.double(), beta.double(), c["eps"]))


@pytest.mark.parametrize("dev", _devices(0))
@pytest.mark.parametrize("c", LN_CASES, ids=_lid)
def test_layernorm(c, dev):
    b = _build_ln(c, dev)
    rows, C = c["rows"], c["C"]
    fn = ops_emulator.layernorm if dev == "cpu" else ops.layernorm
    run = lambda: fn(b["x"], b["y"], b["gamma"], b["beta"], rows=rows, C=C, eps=c["eps"], ldx=b["ldx"], ldy=b["ldy"])
    n0 = ops.launch_count()
    run()
    window = b["y"][:rows, :C]
    what = f"layernorm {_lid(c)} kMaxVec {_kmaxvec(C)}"
    if dev == "cuda":
        assert ops.launch_count() == n0 + 1
        _LN_RAN.add(("layernorm", _kmaxvec(C)))
        first = window.clone()
        window.view(torch.int16).fill_(SENTINEL)
        run()
        assert torch.equal(first.view(torch.int16), window.view(torch.int16)), f"{what}: differs run to run"
    _check_outside(b["ybuf"], window, _sentinel(*b["ybuf"].shape, dev="cpu"), what)
    _close(window.cpu(), b["ref"], what, ns_max=0.0)


STAT_BITS = 0x5A5A5A5A       # fp32 sentinel of the statistics buffer


@pytest.mark.parametrize("dev", _devices(0))
@pytest.mark.parametrize("c", LN_CASES, ids=_lid)
def test_row_stats(c, dev):
    """(mean, rstd) per row against float64: the mean within the rounding of a 64-term lane sum plus the 5-level warp
    tree (80 u of the mean |x|), rstd within 1e-5 relative (the variance is taken about the mean, from registers)."""
    b = _build_ln(c, dev)
    rows, C = c["rows"], c["C"]
    sbuf = torch.full((rows + 2, 2), STAT_BITS, dtype=torch.int32, device=dev).view(torch.float32)
    before = sbuf.cpu().clone()
    fn = ops_emulator.row_stats if dev == "cpu" else ops.row_stats
    run = lambda: fn(b["x"], sbuf[1:], rows=rows, C=C, eps=c["eps"], ldx=b["ldx"])
    n0 = ops.launch_count()
    run()
    what = f"row_stats {_lid(c)} kMaxVec {_kmaxvec(C)}"
    st = sbuf[1:1 + rows].cpu().clone()
    if dev == "cuda":
        assert ops.launch_count() == n0 + 1
        _LN_RAN.add(("row_stats", _kmaxvec(C)))
        sbuf[1:1 + rows].view(torch.int32).fill_(STAT_BITS)
        run()
        assert torch.equal(st.view(torch.int32), sbuf[1:1 + rows].cpu().view(torch.int32)), f"{what}: differs run to run"
    out = sbuf.cpu().view(torch.int32)
    assert torch.equal(out[0], before.view(torch.int32)[0]) and torch.equal(out[-1], before.view(torch.int32)[-1]), \
        f"{what}: wrote outside rows [0, rows)"
    x64 = b["x64"]
    mean, var = x64.mean(1), x64.var(1, unbiased=False)
    rstd = (var + c["eps"]).rsqrt()
    st = st.double()
    assert torch.isfinite(st).all(), what
    dm = (st[:, 0] - mean).abs().max().item()
    tol_m = 80 * 2.0 ** -24 * x64.abs().mean(1).max().item() + 1e-7
    dr = ((st[:, 1] - rstd).abs() / rstd).max().item()
    print(f"{what}: mean err {dm:.2e} (bound {tol_m:.2e}), rstd rel err {dr:.2e}")
    assert dm <= tol_m, f"{what}: mean error {dm:.3e} > {tol_m:.3e}"
    assert dr <= 1e-5, f"{what}: rstd relative error {dr:.3e}"


def test_layernorm_case_table():
    assert {_kmaxvec(C) for C in LN_C} == {2, 5, 8}
    for kv, lo, hi in ((2, 8, 512), (5, 520, 1280), (8, 1288, 2048)):
        assert lo in LN_C and hi in LN_C and _kmaxvec(lo) == _kmaxvec(hi) == kv
    assert {c["rows"] % 8 for c in LN_CASES} >= {0, 1, 7}


# ================================================================================================ refused arguments
REFUSED = ["gn_misaligned_x", "gn_misaligned_y", "gn_ldx_narrow", "gn_ldy_narrow", "ln_misaligned_x", "ln_misaligned_y",
           "ln_ldx_narrow", "ln_ldy_narrow", "rs_misaligned_x", "rs_misaligned_stats", "rs_ldx_narrow"]


@pytest.mark.gpu
@pytest.mark.parametrize("form", REFUSED)
def test_refused_launch_arguments(form):
    """tc_groupnorm, tc_layernorm and tc_row_stats refuse these forms before launching anything
    (include/tooncrafter_b200.h)."""
    from tooncrafter_b200 import _lib
    dev = "cuda"
    rows, C = 64, 256
    x = torch.zeros(rows + 1, C + 16, dtype=torch.float16, device=dev)
    y = torch.zeros(rows + 1, C + 16, dtype=torch.float16, device=dev)
    gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    stats = torch.zeros(rows + 1, 2, device=dev)
    ld = C + 16
    n0 = ops.launch_count()
    with pytest.raises(_lib.TcError, match="tc_groupnorm|tc_layernorm|tc_row_stats"):
        if form.startswith("gn"):
            kw = dict(frames=2, frames_per_stat=1, hw=rows // 2, C=C, ldx=ld, ldy=ld)
            if form == "gn_misaligned_x":
                kw["x_offset"] = 4
            elif form == "gn_misaligned_y":
                kw["y_offset"] = 12
            elif form == "gn_ldx_narrow":
                kw["ldx"] = C - 8
            else:
                kw["ldy"] = C - 64
            ops.groupnorm(x, y, gamma, beta, **kw)
        elif form.startswith("ln"):
            xv, yv, ldx, ldy = x, y, ld, ld
            if form == "ln_misaligned_x":
                xv = x[:, 4:]
            elif form == "ln_misaligned_y":
                yv = y[:, 2:]
            elif form == "ln_ldx_narrow":
                ldx = C - 8
            else:
                ldy = 128
            ops.layernorm(xv, yv, gamma, beta, rows=rows, C=C, ldx=ldx, ldy=ldy)
        else:
            xv, sv, ldx = x, stats, ld
            if form == "rs_misaligned_x":
                xv = x[:, 4:]
            elif form == "rs_misaligned_stats":
                sv = stats.view(-1)[1:]
            else:
                ldx = C - 8
            ops.row_stats(xv, sv, rows=rows, C=C, ldx=ldx)
    assert ops.launch_count() == n0, "a refused launch still launched"
    print(f"{form}: {_lib.load().tc_last_error().decode()}")


@pytest.mark.gpu
def test_matrix_ran_every_norm_path(request):
    """Last in the file: the CUDA cases above ran fused cluster sizes 1..8 and the two-pass path, and kMaxVec 2, 5 and 8
    for both LayerNorm and row_stats."""
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node
            and getattr(it, "callspec", None) is not None and it.callspec.params.get("dev", "cuda") == "cuda"]
    expected = len(GN_CASES) + 2 * len(LN_CASES) + len(REFUSED)
    if len(mine) != expected:
        pytest.skip(f"{len(mine)} of the {expected} CUDA cases were selected")
    print("GroupNorm paths:", sorted(_GN_RAN), "LayerNorm / row_stats:", sorted(_LN_RAN))
    assert _GN_RAN == {("fused", cs) for cs in range(1, 9)} | {("two",)}
    assert _LN_RAN == {(k, v) for k in ("layernorm", "row_stats") for v in (2, 5, 8)}
