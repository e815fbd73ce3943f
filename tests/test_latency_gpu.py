"""Latency mode: two GPUs share one clip, each evaluates one classifier-free-guidance branch per DDIM step
and the predictions are all-gathered.  The result must equal the single-GPU fused path (same algorithm, B = 1 + B = 1
instead of one B = 2 forward).  The NCCL variant needs 2 GPUs (skipped on a single-GPU box, run with `gpurun --gpus 2`);
the single-GPU variant runs the SAME two-rank protocol with both ranks time-sharing cuda:0 over gloo (collectives staged
through host memory), so the pair logic — branch split, per-step exchange, state synchronisation — is exercised wherever
the GPU tests run."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from distributed_harness import LATENCY_BOUND, spawn  # noqa: E402


def _worker(rank, world, one_gpu=False):
    import torch.distributed as dist
    dev = torch.device("cuda", 0 if one_gpu else rank)
    torch.cuda.set_device(dev)
    if one_gpu:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    else:
        dist.init_process_group("nccl", device_id=dev)
    from make_golden import SEED, golden_inputs
    from tiny_config import model_config
    from tooncrafter_b200 import diffusion, synthetic
    from tooncrafter_b200.distributed import latency_pairs
    from tooncrafter_b200.sampler import DDIMSampler
    m = diffusion.instantiate_from_config(model_config())
    synthetic.fill_module_(m, seed=SEED)
    m.perframe_ae = True
    m = m.to(dev).eval()
    gi = golden_inputs()
    to = lambda c: {k: [t.to(dev) for t in v] for k, v in c.items()}
    kw = dict(S=gi["S"], batch_size=1, shape=list(gi["x_T"].shape[1:]), conditioning=to(gi["cond"]),
              unconditional_conditioning=to(gi["uncond"]), eta=1.0, unconditional_guidance_scale=7.5,
              x_T=gi["x_T"].to(dev), fs=gi["fs"].to(dev), timestep_spacing="uniform_trailing", guidance_rescale=0.7,
              verbose=False)
    group, pair, in_pair = latency_pairs()
    torch.manual_seed(1234 + rank)            # deliberately different: the sampler must synchronise the pair itself
    s = DDIMSampler(m)
    s.latency_group = group
    lat, _ = s.sample(**kw)
    both = [torch.empty_like(lat.cpu()) for _ in range(world)]
    if one_gpu:
        dist.all_gather(both, lat.cpu())
    else:
        both = [torch.empty_like(lat) for _ in range(world)]
        dist.all_gather(both, lat)
    res = None
    if rank == 0:
        torch.manual_seed(1234)               # pair-rank 0's stream is the one the pair used
        ref, _ = DDIMSampler(m).sample(**kw)
        res = dict(pair_equal=bool(torch.equal(both[0], both[1])), err=float((lat - ref).abs().max()),
                   scale=float(ref.abs().max()), finite=bool(torch.isfinite(lat).all()))
    dist.barrier()
    dist.destroy_process_group()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("one_gpu", [True, False], ids=["two_ranks_on_one_gpu_gloo", "two_gpus_nccl"])
def test_latency_mode_matches_single_gpu_fused_path(one_gpu):
    if not one_gpu and torch.cuda.device_count() < 2:
        pytest.skip("the NCCL variant pairs two GPUs")
    res = spawn(_worker, one_gpu, world=2, timeout=600)[0]
    print("latency mode vs single-GPU fused path:", res)
    assert res["finite"] and res["pair_equal"], res
    # The B = 1 and B = 2 programs may pick different tiles and k-slices (split-K): fp32 summation order differs, fp16
    # roundings flip, and four free-running DDIM steps amplify that (measured 1.3 % of the scale with split-K on, exactly 0
    # with TC_GEMM_KSPLIT=1, when both programs reduce in the same order).  The bound is of the order of the fp16-vs-fp32
    # error the 4-step golden test accepts for the same sample; a wrong branch / state exchange is O(scale).
    assert res["err"] <= LATENCY_BOUND * res["scale"], res
