"""Conformance matrix of the attention kernels: tc_attention (all five flash_attn_kernel instances it launches),
tc_attention_wide (the 64-, 128- and 256-column value-chunk instances), tc_temporal_attention (the mma.sync kernel for
T <= 16 and the 32-lane kernel above) and tc_softmax_rows, each against a float64 reference of the same operation on
the same fp16-rounded inputs.

Every CUDA case also checks
  * the path that ran: the flash instance (kDV, two segments, causal) follows from (head dim, segments, causal, value
    chunk) and is asserted in the case table; the temporal kernel from T;
  * write bounds: the output is a window of a wider buffer (row stride above the width, a non-zero column offset, rows
    before and after) prefilled with a sentinel bit pattern that must be intact afterwards;
  * read bounds: operand memory outside the views is NaN (columns past a row's view, rows past Lq / Lk / the last token
    in the same allocation), so a read outside a view shows up as a NaN in the result;
  * determinism: a second launch gives a bitwise identical output.

Tolerance against float64, with the bounds of the existing tests of the same paths (tests/test_kernels_gpu.py):
  * P split into fp16 hi + lo parts for the PV product (at most 512 keys per query row, and temporal attention): no
    element outside rtol 1e-3 / atol 1e-4 (ns_max = 0);
  * P rounded to fp16 (more keys): at most 0.1 % of the elements outside it (ns_max = 1e-3), 0.2 % with a growing row
    maximum (test_attention_wide_growing_maximum);
  * the max-norm bound of _close everywhere.

Each case runs twice: on the H100 (marked gpu) and on CPU through tests/ops_emulator.py (tests/clip_emulator.py for head
dim 80 and causal masking), which exercises the case builders, poison and references without a GPU.
"""
import sys
import zlib
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

import clip_emulator  # noqa: E402
import ops_emulator  # noqa: E402
from test_kernels_gpu import _close  # noqa: E402

from tooncrafter_b200 import ops  # noqa: E402

DEVICES = [pytest.param("cpu", id="cpu"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]
GPU_ONLY = [pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]
SENTINEL = 0x5A5A                            # fp16 203.25: bit pattern of untouched output memory
NAN16 = 0x7E00                               # fp16 NaN: bit pattern of the unread gaps of an in-place buffer

_RAN = set()          # flash instances (kDV, two_seg, causal) of every checked CUDA launch
_TEMPORAL_RAN = set()  # "mma" / "lanes" for every checked CUDA temporal launch


def _seed(cid):
    return torch.Generator().manual_seed(zlib.crc32(cid.encode()))


def _nan16(*s, dev):
    return torch.full(s, float("nan"), dtype=torch.float16, device=dev)


def _sentinel(*s, dev, bits=SENTINEL):
    return torch.full(s, bits, dtype=torch.int16, device=dev).view(torch.float16)


def _check_outside(buf, window, what, bits=SENTINEL):
    """Every element of `buf` outside `window` (a view into it) still holds `bits`."""
    flat = buf.view(torch.int16).cpu().reshape(-1)
    keep = torch.ones_like(flat, dtype=torch.bool)
    idx = torch.as_strided(torch.arange(buf.numel()), window.shape, window.stride(),
                           window.storage_offset() - buf.storage_offset())
    keep[idx.reshape(-1)] = False
    bad = ((flat != bits) & keep).nonzero()
    assert bad.numel() == 0, f"{what}: wrote outside the output window ({bad.numel()} elements, first at {bad[0].item()})"


def _ref_attn(q, k, v, scale, causal=False):
    """float64 softmax(q k^T * scale) v over [..., L, d]; causal masks key j for query i when j > i."""
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(s.shape[-2], s.shape[-1], dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    return s.softmax(-1) @ v


# ================================================================================================ tc_attention
def acase(B, Lq, Lk, heads, d=64, causal=False, kv_div=None, layout="sep", amp=1.0, growing=False):
    """Lk: one key count per segment; kv_div likewise (default 1).  layout: sep (q, k, v in separate buffers with
    padded rows) or fused (q / k / v channel slices of one [tokens][3C + 8] tensor, self attention)."""
    Lk = tuple(Lk) if isinstance(Lk, (tuple, list)) else (Lk,)
    kv_div = tuple(kv_div) if kv_div else (1,) * len(Lk)
    return dict(B=B, Lq=Lq, Lk=Lk, heads=heads, d=d, causal=causal, kv_div=kv_div, layout=layout, amp=amp,
                growing=growing)


def _aid(c):
    p = [f"B{c['B']}", f"Lq{c['Lq']}", "Lk" + "+".join(map(str, c["Lk"])), f"h{c['heads']}", f"d{c['d']}", c["layout"]]
    if any(x > 1 for x in c["kv_div"]):
        p.append("div" + "+".join(map(str, c["kv_div"])))
    p += [k for k in ("causal", "growing") if c[k]]
    if c["amp"] != 1.0:
        p.append(f"amp{c['amp']}")
    return "-".join(p)


def _instance(c):
    """(kDV, two-segment, causal) of the flash_attn_kernel instance tc_attention launches (launch_flash)."""
    if c["d"] == 80:
        return (80, False, c["causal"])
    if c["causal"]:
        return (64, False, True)
    return (64, len(c["Lk"]) == 2, False)


def _build_attn(c, dev):
    g = _seed(_aid(c))
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    B, Lq, heads, d = c["B"], c["Lq"], c["heads"], c["d"]
    C = heads * d
    scale = d ** -0.5
    q16 = (rnd(B, Lq, C) * c["amp"]).half()
    segs16 = []
    for Lk, div in zip(c["Lk"], c["kv_div"]):
        kvb = -(-B // div)
        k = rnd(kvb, Lk, C) * c["amp"]
        if c["growing"]:        # later key tiles raise the row maximum
            k = k * torch.linspace(0.2, 3.0, Lk, dtype=torch.float64)[None, :, None]
        segs16.append((k.half(), rnd(kvb, Lk, C).half(), Lk, div))
    kw = dict(q_batches=B, Lq=Lq, heads=heads, scale=scale)
    if d == 80 or c["causal"]:
        kw.update(head_dim=d, causal=c["causal"])
    segs = []
    if c["layout"] == "fused":
        assert len(segs16) == 1 and segs16[0][2] == Lq and segs16[0][3] == 1
        ld = 3 * C + 8
        qkv = _nan16(B * Lq + 3, ld, dev=dev)
        k16, v16 = segs16[0][0], segs16[0][1]
        for i, t in enumerate((q16, k16, v16)):
            qkv[:B * Lq, i * C:(i + 1) * C] = t.reshape(B * Lq, C).to(dev)
        q, kw["ldq"], kw["q_offset"] = qkv, ld, 0
        segs.append(dict(k=qkv, v=qkv, ldk=ld, ldv=ld, Lk=Lq, k_offset=C, v_offset=2 * C))
    else:
        ldq = C + 24
        q = _nan16(B * Lq + 3, ldq, dev=dev)
        q[:B * Lq, 8:8 + C] = q16.reshape(B * Lq, C).to(dev)
        kw.update(ldq=ldq, q_offset=8)
        for i, (k16, v16, Lk, div) in enumerate(segs16):
            kvb = k16.shape[0]
            ldk, ldv = C + 8 * (i + 1), C + 40
            kb, vb = _nan16(kvb * Lk + 2, ldk, dev=dev), _nan16(kvb * Lk + 5, ldv, dev=dev)
            kb[:kvb * Lk, :C] = k16.reshape(-1, C).to(dev)
            vb[:kvb * Lk, 16:16 + C] = v16.reshape(-1, C).to(dev)
            segs.append(dict(k=kb, v=vb, ldk=ldk, ldv=ldv, Lk=Lk, kv_div=div, v_offset=16))
    ldo = C + 16
    out = _sentinel(B * Lq + 2, ldo, dev=dev)
    kw.update(ldo=ldo, out_offset=ldo + 8)       # one row before the window, 8 columns in
    window = out[1:1 + B * Lq, 8:8 + C]
    sp = lambda t: t.double().reshape(t.shape[0], t.shape[1], heads, d).transpose(1, 2)
    ref = torch.zeros(B, heads, Lq, d, dtype=torch.float64)
    for k16, v16, Lk, div in segs16:
        idx = torch.arange(B) // div
        ref += _ref_attn(sp(q16), sp(k16)[idx], sp(v16)[idx], scale, c["causal"])
    ref = ref.transpose(1, 2).reshape(B * Lq, C)
    return dict(q=q, segs=segs, out=out, kw=kw, window=window, ref=ref)


def _launch_attn(c, b, dev):
    if dev == "cpu":
        fn = clip_emulator.attention if "head_dim" in b["kw"] else ops_emulator.attention
        fn(b["q"], b["segs"], b["out"], **b["kw"])
        return
    n0 = ops.launch_count()
    ops.attention(b["q"], b["segs"], b["out"], **b["kw"])
    assert ops.launch_count() == n0 + 1
    _RAN.add(_instance(c))


def _attn_tol(keys, growing=False):
    """keys: the most keys one query row sees (launch_flash splits P when it is <= 512)."""
    if keys <= 512:
        return 0.0            # P split into hi + lo: only the output rounding is left
    # P rounded to fp16 for the PV product (as test_attention_self); a growing maximum as test_attention_wide_growing_maximum
    return 2e-3 if growing else 1e-3


def _run_twice(launch, b, dev):
    launch()
    if dev == "cuda":
        first = b["window"].clone()
        b["window"].view(torch.int16).fill_(SENTINEL)
        launch()
        assert torch.equal(first.view(torch.int16), b["window"].view(torch.int16)), "output differs run to run"


ATTN_LS = (1, 63, 64, 65, 127, 512, 513, 1100)
ATTN_CASES = (
    # one segment, head dim 64: Lq != Lk over the tile edges and both sides of the split_p switch at 512 keys
    [acase(2, lq, lk, h) for lq, lk, h in ((1, 63, 1), (63, 64, 2), (64, 65, 3), (65, 127, 4), (127, 512, 5),
                                            (512, 513, 6), (513, 1100, 7), (1100, 1, 8), (1, 1100, 9), (65, 512, 10))]
    + [acase(3, 127, 127, 2, layout="fused"), acase(2, 513, 513, 5, layout="fused"), acase(1, 1, 1, 1, layout="fused")]
    + [acase(6, 65, 77, 4, kv_div=(3,)), acase(4, 200, 1100, 2, kv_div=(4,))]
    # two segments (text shared by kv_div query batches + per-batch image), one on each side of 512 keys
    + [acase(4, 160, (77, 16), 5, kv_div=(2, 1)), acase(4, 127, (513, 64), 3, kv_div=(4, 1)),
       acase(2, 65, (100, 1100), 2), acase(3, 1, (512, 1), 1, kv_div=(3, 1))]
    # causal, Lq < Lk and Lq > Lk; head dim 80 with and without the mask
    + [acase(2, 63, 127, 4, causal=True), acase(2, 513, 65, 3, causal=True), acase(1, 77, 77, 20, causal=True),
       acase(2, 1100, 1100, 1, causal=True)]
    + [acase(2, 257, 257, 16, d=80), acase(1, 65, 513, 2, d=80), acase(3, 1, 63, 5, d=80), acase(2, 1100, 1100, 1, d=80),
       acase(2, 77, 77, 4, d=80, causal=True), acase(1, 127, 64, 3, d=80, causal=True),
       acase(1, 65, 1100, 2, d=80, causal=True)]
    # score range: large |scale q k|, and keys whose scores grow along the sequence (each head dim and form)
    + [acase(2, 200, 300, 2, amp=4.0), acase(1, 130, 1100, 2, amp=4.0), acase(2, 130, 1100, 2, growing=True),
       acase(2, 130, 300, 2, growing=True), acase(2, 200, 1100, 2, d=80, growing=True),
       acase(1, 300, 300, 2, causal=True, growing=True), acase(2, 100, (1100, 77), 2, growing=True)]
)


def test_attention_case_table():
    """The table covers what the issue of each instance needs (no launch)."""
    assert {_instance(c) for c in ATTN_CASES} == {(64, False, False), (64, True, False), (64, False, True),
                                                  (80, False, False), (80, False, True)}
    lengths = {c["Lq"] for c in ATTN_CASES} | {lk for c in ATTN_CASES for lk in c["Lk"]}
    assert set(ATTN_LS) <= lengths
    assert {c["heads"] for c in ATTN_CASES} >= set(range(1, 11))
    assert any(len(c["Lk"]) == 2 and min(c["Lk"]) <= 512 < max(c["Lk"]) for c in ATTN_CASES)
    assert any(c["causal"] and c["Lq"] < c["Lk"][0] for c in ATTN_CASES)
    assert any(c["causal"] and c["Lq"] > c["Lk"][0] for c in ATTN_CASES)
    for c in ATTN_CASES:
        assert c["d"] == 64 or len(c["Lk"]) == 1


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", ATTN_CASES, ids=_aid)
def test_attention(c, dev):
    b = _build_attn(c, dev)
    _run_twice(lambda: _launch_attn(c, b, dev), b, dev)
    _check_outside(b["out"], b["window"], _aid(c))
    keys = min(c["Lq"], max(c["Lk"])) if c["causal"] else max(c["Lk"])      # the most keys one query row sees
    what = f"{_aid(c)} instance {_instance(c)} split_p {keys <= 512}"
    _close(b["window"].cpu(), b["ref"], what, ns_max=_attn_tol(keys, c["growing"]))


# ================================================================================================ tc_attention_wide
def wcase(B, Lq, Lk, D, growing=False, fused=False):
    return dict(B=B, Lq=Lq, Lk=Lk, D=D, growing=growing, fused=fused)


def _wid(c):
    return f"wide-B{c['B']}-Lq{c['Lq']}-Lk{c['Lk']}-D{c['D']}" + ("-growing" if c["growing"] else "") + (
        "-fused" if c["fused"] else "")


def _wide_instance(D):
    return (256 if D % 256 == 0 else 128 if D % 128 == 0 else 64, False, False)


def _wide_cpu(q, k, v, ldq, ldk, ldv, out, ldo, batches, Lq, Lk, D, scale):
    """fp32 emulation of the tc_attention_wide ABI on [batches][L][D] views with the given row strides."""
    st = ops_emulator._strided
    Q = st(q, (batches, Lq, D), (Lq * ldq, ldq, 1)).float()
    K = st(k, (batches, Lk, D), (Lk * ldk, ldk, 1)).float()
    V = st(v, (batches, Lk, D), (Lk * ldv, ldv, 1)).float()
    st(out, (batches, Lq, D), (Lq * ldo, ldo, 1)).copy_((((Q @ K.transpose(-1, -2)) * scale).softmax(-1) @ V).half())


def _build_wide(c, dev):
    g = _seed(_wid(c))
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    B, Lq, Lk, D = c["B"], c["Lq"], c["Lk"], c["D"]
    q16 = rnd(B, Lq, D).half()
    k = rnd(B, Lk, D)
    if c["growing"]:
        k = k * torch.linspace(0.2, 3.0, Lk, dtype=torch.float64)[None, :, None]
    k16, v16 = k.half(), rnd(B, Lk, D).half()
    ldo = D + 24
    out = _sentinel(B * Lq + 2, ldo, dev=dev)
    window = out[1:1 + B * Lq, 16:16 + D]
    if c["fused"]:
        assert Lq == Lk
        ld = 3 * D + 8
        qkv = _nan16(B * Lq + 2, ld, dev=dev)
        for i, t in enumerate((q16, k16, v16)):
            qkv[:B * Lq, i * D:(i + 1) * D] = t.reshape(-1, D).to(dev)
        ops_args = (qkv, ld)
        views = None
    else:
        ldq, ldk, ldv = D + 8, D + 16, D + 64
        qb, kb, vb = _nan16(B * Lq + 1, ldq, dev=dev), _nan16(B * Lk + 3, ldk, dev=dev), _nan16(B * Lk + 1, ldv, dev=dev)
        qb[:B * Lq, 8:8 + D] = q16.reshape(-1, D).to(dev)
        kb[:B * Lk, :D] = k16.reshape(-1, D).to(dev)
        vb[:B * Lk, 64:64 + D] = v16.reshape(-1, D).to(dev)
        views = (qb[:, 8:], kb, vb[:, 64:], ldq, ldk, ldv)
        ops_args = None
    ref = _ref_attn(q16.double(), k16.double(), v16.double(), D ** -0.5).reshape(B * Lq, D)
    return dict(out=out, window=window, ref=ref, views=views, ops_args=ops_args)


def _launch_wide(c, b, dev):
    B, Lq, Lk, D = c["B"], c["Lq"], c["Lk"], c["D"]
    scale = D ** -0.5
    w = b["window"]
    if b["ops_args"] is not None:
        qkv, ld = b["ops_args"]
        fn = ops_emulator.attention_wide if dev == "cpu" else ops.attention_wide
        n0 = ops.launch_count()
        fn(qkv, b["out"], batches=B, L=Lq, D=D, scale=scale, ld=ld, ldo=w.stride(0), q_offset=0, k_offset=D,
           v_offset=2 * D, out_offset=w.storage_offset() - b["out"].storage_offset())
    else:
        # through the C ABI: ops.attention_wide passes one L for Lq and Lk
        q, k, v, ldq, ldk, ldv = b["views"]
        if dev == "cpu":
            _wide_cpu(q, k, v, ldq, ldk, ldv, w, w.stride(0), B, Lq, Lk, D, scale)
            return
        from tooncrafter_b200 import _lib
        n0 = ops.launch_count()
        _lib.check(_lib.load().tc_attention_wide(q.data_ptr(), k.data_ptr(), v.data_ptr(), ldq, ldk, ldv, w.data_ptr(),
                                                 w.stride(0), B, Lq, Lk, D, scale, ops._stream()), "tc_attention_wide")
    if dev == "cuda":
        assert ops.launch_count() == n0 + 1
        _RAN.add(_wide_instance(D))


WIDE_DS = (64, 128, 192, 256, 384, 512)
WIDE_CASES = ([wcase(2, 130, 130, D) for D in WIDE_DS]                                        # ragged L
              + [wcase(1, 65, 1100, D) for D in WIDE_DS]                                      # Lq < Lk, P rounded
              + [wcase(2, 513, 63, D) for D in (64, 192, 512)]                                # Lq > Lk
              + [wcase(2, 1, 512, 384), wcase(1, 127, 513, 256)]
              + [wcase(2, 300, 300, D, fused=True) for D in (128, 512)]                       # the VAE's fused qkv
              + [wcase(1, 200, 1024, D, growing=True) for D in (64, 128, 512)])


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", WIDE_CASES, ids=_wid)
def test_attention_wide(c, dev):
    b = _build_wide(c, dev)
    _run_twice(lambda: _launch_wide(c, b, dev), b, dev)
    _check_outside(b["out"], b["window"], _wid(c))
    _close(b["window"].cpu(), b["ref"], f"{_wid(c)} instance {_wide_instance(c['D'])}",
           ns_max=_attn_tol(c["Lk"], c["growing"]))


# ================================================================================================ tc_temporal_attention
def tcase(B, T, P, heads):
    return dict(B=B, T=T, P=P, heads=heads)


def _tid(c):
    return f"temporal-B{c['B']}-T{c['T']}-P{c['P']}-h{c['heads']}"


def _build_temporal(c, dev):
    g = _seed(_tid(c))
    B, T, P, heads = c["B"], c["T"], c["P"], c["heads"]
    C = heads * 64
    rows = B * T * P
    x16 = torch.randn(B, T, P, 3 * C, generator=g).half()
    ld = 3 * C + 8
    qkv = _nan16(rows + 2, ld, dev=dev)
    qkv[:rows, :3 * C] = x16.reshape(rows, 3 * C).to(dev)
    ldo = C + 8
    out = _sentinel(rows + 2, ldo, dev=dev)
    window = out[1:1 + rows, :C]
    xs = x16.to(dev).double().permute(0, 2, 1, 3).reshape(B * P, T, 3, heads, 64).permute(2, 0, 3, 1, 4)   # [3][BP][h][T][64]
    ref = _ref_attn(xs[0], xs[1], xs[2], 64 ** -0.5)                                               # [BP][h][T][64]
    ref = ref.permute(0, 2, 1, 3).reshape(B, P, T, C).permute(0, 2, 1, 3).reshape(rows, C).cpu()
    return dict(qkv=qkv, ld=ld, out=out, window=window, ref=ref)


def _launch_temporal(c, b, dev):
    C = c["heads"] * 64
    kw = dict(ld=b["ld"], ldo=b["window"].stride(0), B=c["B"], T=c["T"], P=c["P"], heads=c["heads"], scale=64 ** -0.5,
              q_offset=0, k_offset=C, v_offset=2 * C)
    if dev == "cpu":
        ops_emulator.temporal_attention(b["qkv"], b["qkv"], b["qkv"], b["out"][1:], **kw)
        return
    n0 = ops.launch_count()
    ops.temporal_attention(b["qkv"], b["qkv"], b["qkv"], b["out"][1:], **kw)
    assert ops.launch_count() == n0 + 1
    _TEMPORAL_RAN.add("mma" if c["T"] <= 16 else "lanes")


def _mma_warps():
    """Warps of the grid-stride temporal_attn_mma_kernel: 16 blocks of 4 warps per SM."""
    return 16 * 4 * torch.cuda.get_device_properties(0).multi_processor_count


TEMPORAL_CASES = [tcase(1 + t % 3, t, 7 + 13 * t, 1 + t % 10) for t in range(1, 33)]      # every T, ragged P
BIG_TEMPORAL = [tcase(2, 9, 1300, 10), tcase(3, 2, 2900, 3), tcase(1, 32, 300, 10)]       # mma: >= 3 items per warp


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", TEMPORAL_CASES, ids=_tid)
def test_temporal_attention(c, dev):
    b = _build_temporal(c, dev)
    _run_twice(lambda: _launch_temporal(c, b, dev), b, dev)
    _check_outside(b["out"], b["window"], _tid(c))
    # P split into fp16 hi + lo parts in both kernels (the 32-lane kernel keeps P in fp32)
    _close(b["window"].cpu(), b["ref"], f"{_tid(c)} ({'mma' if c['T'] <= 16 else 'lanes'})", ns_max=0.0)


@pytest.mark.parametrize("dev", GPU_ONLY)
@pytest.mark.parametrize("c", BIG_TEMPORAL, ids=_tid)
def test_temporal_attention_grid_stride(c, dev):
    """More items than three times the mma kernel's warps: every warp runs several items and reuses its V tile."""
    if c["T"] <= 16:
        assert c["B"] * c["P"] * c["heads"] >= 3 * _mma_warps()
    test_temporal_attention(c, dev)


# ================================================================================================ tc_softmax_rows
def scase(rows, cols, lds, scale, spread=3.0):
    return dict(rows=rows, cols=cols, lds=lds, scale=scale, spread=spread)


def _sid(c):
    return f"softmax-{c['rows']}x{c['cols']}-lds{c['lds']}-scale{c['scale']}-spread{c['spread']}"


SOFTMAX_CASES = ([scase(5, cols, cols, 0.125) for cols in (1, 7, 100, 255, 256, 257, 1000)]
                 + [scase(300, 2560, 2560, 0.125), scase(7, 2561, 2600, 0.125), scase(3, 4000, 4040, 0.5)]
                 + [scase(9, 33, 48, 1.0), scase(4, 300, 320, -0.25)]
                 # wide spread: |scale| * (max - min) well past 88 (exp overflow of a raw-maximum form for scale < 0)
                 + [scase(6, 1000, 1008, 1.0, spread=60.0), scase(6, 1000, 1008, -1.0, spread=60.0),
                    scase(3, 2561, 2568, -0.7, spread=200.0), scase(2, 200, 200, -2.0, spread=100.0)])


def _build_softmax(c, dev):
    g = _seed(_sid(c))
    rows, cols, lds = c["rows"], c["cols"], c["lds"]
    x16 = (torch.randn(rows, cols, generator=g, dtype=torch.float64) * c["spread"]).half()
    buf = _sentinel(rows + 2, lds, dev=dev, bits=NAN16)      # gaps and the rows around the window: NaN
    window = buf[1:1 + rows, :cols]
    window.copy_(x16.to(dev))
    ref = (x16.double() * c["scale"]).softmax(-1)
    return dict(buf=buf, window=window, ref=ref, x16=x16)


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("c", SOFTMAX_CASES, ids=_sid)
def test_softmax_rows(c, dev):
    b = _build_softmax(c, dev)
    fn = ops_emulator.softmax_rows if dev == "cpu" else ops.softmax_rows
    fn(b["buf"][1:], rows=c["rows"], cols=c["cols"], scale=c["scale"], lds=c["lds"])
    if dev == "cuda":
        first = b["window"].clone()
        b["window"].copy_(b["x16"].to(dev))
        fn(b["buf"][1:], rows=c["rows"], cols=c["cols"], scale=c["scale"], lds=c["lds"])
        assert torch.equal(first.view(torch.int16), b["window"].view(torch.int16)), "output differs run to run"
    _check_outside(b["buf"], b["window"], _sid(c), bits=NAN16)
    _close(b["window"].cpu(), b["ref"], _sid(c), rel=2e-3, abs_=1e-5)     # the bounds of test_softmax_rows


# ================================================================================================ refused arguments
REFUSED = ["temporal_misaligned_q", "temporal_misaligned_out", "temporal_ld_narrow", "temporal_ldo_narrow",
           "softmax_lds_narrow"]


@pytest.mark.gpu
@pytest.mark.parametrize("form", REFUSED)
def test_refused_launch_arguments(form):
    """tc_temporal_attention and tc_softmax_rows refuse these forms before launching anything
    (include/tooncrafter_b200.h)."""
    from tooncrafter_b200 import _lib
    dev = "cuda"
    B, T, P, heads = 1, 4, 8, 2
    C = heads * 64
    qkv = torch.zeros(B * T * P + 1, 3 * C, dtype=torch.float16, device=dev)
    out = torch.zeros(B * T * P + 1, C, dtype=torch.float16, device=dev)
    kw = dict(ld=3 * C, ldo=C, B=B, T=T, P=P, heads=heads, scale=0.125, q_offset=0, k_offset=C, v_offset=2 * C)
    n0 = ops.launch_count()
    with pytest.raises(_lib.TcError, match="tc_temporal_attention|tc_softmax_rows"):
        if form == "temporal_misaligned_q":
            kw["q_offset"] = 4
        elif form == "temporal_misaligned_out":
            out = out.view(-1)[4:]
        elif form == "temporal_ld_narrow":
            kw.update(ld=C - 8, k_offset=0, v_offset=0)
        elif form == "temporal_ldo_narrow":
            kw["ldo"] = C - 64
        if form.startswith("temporal"):
            ops.temporal_attention(qkv, qkv, qkv, out, **kw)
        else:
            ops.softmax_rows(out, rows=4, cols=C, lds=C - 8, scale=1.0)
    assert ops.launch_count() == n0, "a refused launch still launched"
    print(f"{form}: {_lib.load().tc_last_error().decode()}")


_MATRIX = [ATTN_CASES, WIDE_CASES, TEMPORAL_CASES, SOFTMAX_CASES]


@pytest.mark.gpu
def test_matrix_ran_every_attention_path(request):
    """Last in the file: the CUDA cases above ran all seven flash instances and both temporal kernels."""
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node
            and getattr(it, "callspec", None) is not None and it.callspec.params.get("dev", "cuda") == "cuda"]
    expected = sum(len(t) for t in _MATRIX) + len(BIG_TEMPORAL) + len(REFUSED)
    if len(mine) != expected:
        pytest.skip(f"{len(mine)} of the {expected} CUDA cases were selected")
    print("flash instances:", sorted(_RAN), "temporal kernels:", sorted(_TEMPORAL_RAN))
    assert _RAN == {(64, False, False), (64, True, False), (64, False, True), (80, False, False), (80, False, True),
                    (128, False, False), (256, False, False)}
    assert _TEMPORAL_RAN == {"mma", "lanes"}
