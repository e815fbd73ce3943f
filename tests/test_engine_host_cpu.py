"""CPU host-logic tests: the UNet engine's recorded program (weight packing, slices, strides, tap tables, arena
reuse, program order) is interpreted by tests/ops_emulator.py in plain PyTorch and compared with the reference
golden.  This validates everything EXCEPT the CUDA kernels themselves (tests/test_kernels_gpu.py, -m gpu)."""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

import ops_emulator  # noqa: E402
from make_golden import SEED, golden_inputs  # noqa: E402
from tiny_config import TINY_T, TINY_UNET  # noqa: E402

from tooncrafter_b200 import engine, modules, synthetic  # noqa: E402
from tooncrafter_b200.runtime import Arena  # noqa: E402

GOLD = np.load(HERE / "golden" / "tiny_reference_outputs.npz")


def test_arena_alloc_free_coalesce():
    a = Arena(1 << 20, "cpu")
    offs = [a.alloc(1000) for _ in range(8)]
    assert len(set(offs)) == 8 and all(o % Arena.ALIGN == 0 for o in offs)
    for o in offs[1:7]:
        a.free(o)
    big = a.alloc(6 * 1024)              # the six freed 1 KiB blocks coalesced into one hole
    assert big == offs[1]
    a.free(big); a.free(offs[0]); a.free(offs[7])
    assert a.free_blocks == [(0, 1 << 20)] and a.in_use == 0


def test_unet_program_interpreted_on_cpu_matches_reference_golden():
    m = modules.UNetModel(**TINY_UNET)
    synthetic.fill_module_(m, seed=SEED, prefix="model.diffusion_model.")
    eng = engine.UNetEngine(m.eval(), device="cpu", plan_only=True)
    gi = golden_inputs()["unet"]
    y = eng.forward(gi["x"], gi["t"], gi["ctx"], gi["fs"], executor=ops_emulator.executor)
    ref = torch.from_numpy(GOLD["unet_y"])
    err = (y.float() - ref).abs().max().item()
    assert err < 2e-2 * ref.abs().max().item(), err       # fp16 activation storage in the interpreter
    plan = eng.plan_for(2, TINY_T, 16, 16, gi["ctx"].shape[1])
    assert len(plan.main) > 500 and len(plan.ctx) == 32    # 16 spatial transformers x (text, image) K/V GEMMs
    assert plan.arena.in_use <= plan.arena.high_water <= plan.arena.buf.numel()
    # every block boundary matches its geometry
    for _, name, act in plan.marks:
        assert act.rows * act.C > 0 and act.ld >= act.C


def test_vae_encoder_and_decoder_programs_interpreted_on_cpu_match_reference_golden():
    """Host logic of the two VAE engines (weight packing, tap tables, phase split, reference-context packing, arena
    reuse) without a GPU: their recorded programs run on the PyTorch interpreter against the reference's outputs."""
    from oracle import vae_oracle
    from tiny_config import TINY_DDCONFIG
    from tooncrafter_b200 import diffusion, layout, vae_engine
    ae = diffusion.AutoencoderKL_Dualref(ddconfig=TINY_DDCONFIG, embed_dim=4).eval()
    synthetic.fill_module_(ae, seed=SEED, prefix="first_stage_model.")
    gi = golden_inputs()
    # ---- encoder (+ quant_conv): moments and the five hidden maps
    enc = vae_engine.EncoderEngine(ae, device="cpu", plan_only=True)
    moments, hidden = enc.encode(gi["frames"], executor=ops_emulator.executor)
    gm = torch.from_numpy(GOLD["enc_moments"])
    assert (moments.float() - gm).abs().max().item() < 3e-2 * gm.abs().max().item()
    for i, h in enumerate(hidden):
        sub = torch.from_numpy(GOLD[f"enc_hidden{i}_sub"])
        assert (h.float().flatten()[::97] - sub).abs().max().item() < 3e-2 * sub.abs().max().item() + 1e-2, i
    # ---- decoder, fed with the fp32 oracle's hidden states (as the GPU test does)
    sd = {"first_stage_model." + k: v for k, v in ae.state_dict().items()}
    _, hid32 = vae_oracle.encode_hidden(sd, layout.encoder_layout(TINY_DDCONFIG), gi["frames"])
    ref_ctx = [h.reshape(1, 2, *h.shape[1:]).permute(0, 2, 1, 3, 4).contiguous() for h in hid32]
    zz = (gi["z"].permute(0, 2, 1, 3, 4).reshape(TINY_T, 4, 16, 16) / 0.18215).contiguous()
    dec = vae_engine.DecoderEngine(ae.decoder, device="cpu", plan_only=True)
    y = dec.decode(zz, ref_ctx, executor=ops_emulator.executor)
    gold = torch.from_numpy(GOLD["decode"])[0].permute(1, 0, 2, 3)
    assert (y.float() - gold).abs().max().item() < 3e-2 * gold.abs().max().item() + 1e-2


def _check_conv_gemm_call(a, kw):
    """Preconditions tc_conv_gemm documents / enforces (include/tooncrafter_b200.h, csrc/tc_gemm.cu TC_CHECK_ARG)."""
    a_dims, a_strides, w, taps, out_dims, n_cols = a[1], a[2], a[3], a[4], a[6], a[7]
    assert a_dims[3] > 0 and a_dims[3] % 64 == 0, "C must be a positive multiple of 64"
    assert all(s % 8 == 0 for s in a_strides), "A strides must be multiples of 8 elements"
    assert 1 <= len(taps) <= 9
    assert w.shape[1] == len(taps) * a_dims[3] and w.shape[0] >= n_cols and w.stride(0) % 8 == 0
    geglu = kw.get("geglu", False)
    width = n_cols // 2 if geglu else n_cols
    ldc = kw.get("ldc") or width
    assert ldc % 8 == 0 and ldc >= width and all(d > 0 for d in out_dims) and n_cols > 0
    for off in ("a_offset", "out_offset", "res_offset"):
        assert kw.get(off, 0) % 8 == 0, "16-byte aligned operand slices"
    if geglu:
        bn = kw.get("block_n", 0)
        assert bn > 0 and bn % 64 == 0 and n_cols % bn == 0 and kw.get("res") is None and kw.get("bias2") is None
        assert kw.get("acc_scale", 1.0) == 1.0, "GEGLU takes no acc_scale"
    if kw.get("res") is not None:
        ldr = kw.get("ldr") or n_cols
        assert ldr % 8 == 0 and ldr >= n_cols
    b2 = kw.get("bias2")
    if b2 is not None:
        # read 8 halfs (16 bytes) at a time: aligned base, row stride a multiple of 8
        assert b2.dtype == torch.float16 and b2.stride(0) % 8 == 0 and b2.storage_offset() % 8 == 0
        assert b2.shape[1] >= n_cols and kw.get("bias2_rows_per", 0) > 0
    if kw.get("ln_stats") is not None:
        assert kw.get("ln_u") is not None and n_cols % 16 == 0
        if kw.get("ln_nslots", 0):
            assert len(taps) == 1 and 1 <= kw["ln_nslots"] <= 64
    if kw.get("row_stats") is not None:
        bn = kw.get("block_n", 0)
        assert bn > 0 and bn % 32 == 0 and not geglu and kw["row_stats_slots"] == -(-n_cols // bn)
        assert kw["row_stats"].numel() >= 2 * kw["row_stats_slots"] * out_dims[0] * out_dims[1] * out_dims[2]


def _aligned(t, off=0):
    """16-byte aligned operand: the tensor's element offset plus the op's offset is a multiple of 8 halfs."""
    return (t.storage_offset() + off) % 8 == 0


def _check_norm_attention_call(fn, a, kw):
    """Preconditions tc_groupnorm, tc_layernorm, tc_row_stats, tc_temporal_attention and tc_attention enforce
    (include/tooncrafter_b200.h, TC_CHECK_ARG in csrc/tc_norm.cu and csrc/tc_attn.cu)."""
    from tooncrafter_b200 import ops
    name = fn.__name__
    if fn in (ops.groupnorm, ops.layernorm, ops.row_stats):
        C = kw["C"]
        ldx = kw.get("ldx") or C
        assert C % 8 == 0 and ldx % 8 == 0 and ldx >= C and _aligned(a[0], kw.get("x_offset", 0)), name
        if fn is ops.row_stats:
            assert a[1].storage_offset() % 2 == 0, "row_stats: 8-byte aligned statistics"
        else:
            ldy = kw.get("ldy") or C
            assert ldy % 8 == 0 and ldy >= C and _aligned(a[1], kw.get("y_offset", 0)), name
    elif fn is ops.temporal_attention:
        C = kw["heads"] * 64
        assert kw["ld"] % 8 == 0 and kw["ldo"] % 8 == 0 and kw["ld"] >= C and kw["ldo"] >= C and 0 < kw["T"] <= 32
        for t, off in zip(a, ("q_offset", "k_offset", "v_offset", None)):
            assert _aligned(t, kw.get(off, 0) if off else 0), f"temporal_attention: {off or 'out'} misaligned"
    elif fn is ops.attention:
        q, segs, out = a
        assert kw["ldq"] % 8 == 0 and kw["ldo"] % 8 == 0 and 1 <= len(segs) <= 2
        assert _aligned(q, kw.get("q_offset", 0)) and _aligned(out, kw.get("out_offset", 0))
        for sg in segs:
            assert sg["ldk"] % 8 == 0 and sg["ldv"] % 8 == 0 and sg["Lk"] > 0 and sg.get("kv_div", 1) > 0
            assert _aligned(sg["k"], sg.get("k_offset", 0)) and _aligned(sg["v"], sg.get("v_offset", 0))


def _check_program(calls):
    from tooncrafter_b200 import ops
    seen = set()
    for fn, a, kw in calls:
        if fn is ops.conv_gemm:
            _check_conv_gemm_call(a, kw)
        elif fn in (ops.groupnorm, ops.layernorm, ops.row_stats, ops.temporal_attention, ops.attention):
            _check_norm_attention_call(fn, a, kw)
            seen.add(fn.__name__)
    return seen


def test_programs_plan_for_other_geometries_with_valid_launch_arguments():
    """Planning is pure host logic: build the full-size UNet / VAE programs on the meta device for the 512 and the 1024
    model geometry (configs/training_1024_v1.0: latent 72x128) and a small odd one, and check every recorded tc_conv_gemm
    call against the C ABI's preconditions (no GPU, no memory)."""
    from tiny_config import FULL_DDCONFIG, FULL_UNET
    from tooncrafter_b200 import ops, vae_engine
    with torch.device("meta"):
        unet = modules.UNetModel(**FULL_UNET)
        dec = modules.VideoDecoder(**FULL_DDCONFIG)
    eng = engine.UNetEngine(unet, device="meta", plan_only=True)
    for (B, T, H, W) in ((2, 16, 40, 64), (2, 16, 72, 128), (1, 16, 40, 64), (2, 8, 24, 40)):
        plan = eng.plan_for(B, T, H, W, 77 + 16 * T)
        calls = list(plan.ctx.calls) + list(plan.main.calls)
        gemms = [(a, kw) for fn, a, kw in calls if fn is ops.conv_gemm]
        assert len(plan.main) == 664 and len(gemms) > 400
        assert _check_program(calls) == {"groupnorm", "attention", "temporal_attention"}
        assert plan.arena.high_water < (170 << 30)
    deng = vae_engine.DecoderEngine(dec, device="meta", plan_only=True)
    for (T, h, w) in ((16, 40, 64), (14, 40, 64), (16, 72, 128)):
        plan = deng.plan_for(T, h, w)
        calls = list(plan.ctx.calls) + list(plan.main.calls)
        assert _check_program(calls) == {"groupnorm", "attention"}
        assert plan.arena.high_water < (170 << 30)
        # the mid-block AttnBlock (autoencoder_dualref.py:172-206) is ONE fused launch: head dim = its 512 channels, q / k / v
        # channel slices of one projection output, no score matrix in memory (no softmax_rows, no per-frame score GEMMs)
        wide = [(a, kw) for fn, a, kw in calls if fn is ops.attention_wide]
        assert len(wide) == 1 and not any(fn is ops.softmax_rows for fn, a, kw in calls)
        kw = wide[0][1]
        assert kw["D"] == 512 and kw["batches"] == T and kw["L"] == h * w and kw["ld"] == 3 * 512 and kw["ldo"] == 512
        assert (kw["q_offset"], kw["k_offset"], kw["v_offset"]) == (0, 512, 1024) and abs(kw["scale"] - 512 ** -0.5) < 1e-9


def test_freshly_allocated_contexts_are_never_served_from_a_stale_cache():
    """Regression (round-1 ADVICE, engine.py set_context): callers build the conditioning as a fresh torch.cat
    temporary per call; once the previous one is freed the allocator recycles its address with version 0 and the
    same shape, so nothing pointer-derived identifies the content.  Six successive forwards with different,
    immediately-freed contexts must each equal a forward through a brand-new engine."""
    m = modules.UNetModel(**TINY_UNET)
    synthetic.fill_module_(m, seed=SEED, prefix="model.diffusion_model.")
    m.eval()
    eng = engine.UNetEngine(m, device="cpu", plan_only=True)
    gi = golden_inputs()["unet"]
    seen_ptrs = []
    for k in range(6):
        g = torch.Generator().manual_seed(100 + k)
        ctx = torch.cat([torch.randn(2, 77, gi["ctx"].shape[2], generator=g),
                         torch.randn(2, gi["ctx"].shape[1] - 77, gi["ctx"].shape[2], generator=g)], 1)
        seen_ptrs.append(ctx.data_ptr())
        y = eng.forward(gi["x"], gi["t"], ctx, gi["fs"], executor=ops_emulator.executor).clone()
        fresh = engine.UNetEngine(m, device="cpu", plan_only=True)
        y_ref = fresh.forward(gi["x"], gi["t"], ctx, gi["fs"], executor=ops_emulator.executor)
        assert torch.equal(y, y_ref), f"forward {k} used a stale conditioning"
        del ctx
    # (informational) the scenario is real when the allocator did recycle an address
    print("distinct context addresses over 6 calls:", len(set(seen_ptrs)))


def test_engine_repacks_when_any_parameter_changes():
    """matches() fingerprints every parameter: an in-place edit of a LATE block (not the first tensor) re-packs."""
    m = modules.UNetModel(**TINY_UNET)
    synthetic.fill_module_(m, seed=SEED, prefix="model.diffusion_model.")
    eng = engine.UNetEngine(m.eval(), device="cpu", plan_only=True)
    assert eng.matches(m)
    with torch.no_grad():
        list(m.parameters())[-1].add_(1.0)
    assert not eng.matches(m)


def test_openclip_programs_plan_with_valid_launch_arguments():
    """The full-size OpenCLIP text and image tower programs, planned on the meta device: every tc_conv_gemm,
    tc_layernorm, tc_row_stats and tc_attention call satisfies the C ABI's preconditions."""
    from tooncrafter_b200.cond_engine import ClipImageEngine, ClipTextEngine
    with torch.device("meta"):
        t = modules.FrozenOpenCLIPEmbedder(layer="penultimate")
        i = modules.FrozenOpenCLIPImageEmbedderV2()
    for eng, B in ((ClipTextEngine(t, device="meta", plan_only=True), 2), (ClipImageEngine(i, device="meta", plan_only=True), 2)):
        assert _check_program(list(eng.plan_for(B).main.calls)) == {"layernorm", "row_stats", "attention"}


def test_plan_only_engines_refuse_to_execute_without_an_executor():
    """A plan-only engine's programs hold CPU / meta tensors: without an executor to interpret them, executing raises
    the engines' common error instead of reaching a launch."""
    import pytest
    from make_golden_clip import tiny_image, tiny_pixels, tiny_text, tiny_tokens
    from make_golden_resampler import TINY, tiny_input
    from tooncrafter_b200.cond_engine import ClipImageEngine, ClipTextEngine, ResamplerEngine
    rs = modules.Resampler(**TINY).eval()
    runs = [(ResamplerEngine(rs, device="cpu", plan_only=True), tiny_input()),
            (ClipTextEngine(tiny_text(), device="cpu", plan_only=True), tiny_tokens()),
            (ClipImageEngine(tiny_image(), device="cpu", plan_only=True), tiny_pixels())]
    for eng, x in runs:
        with pytest.raises(RuntimeError, match="plan_only engine cannot execute"):
            eng.forward(x)
