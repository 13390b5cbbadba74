"""GPU: the frame-masked rectified-flow step kernel (osb_rf_masked_step) against an fp32 torch restatement of its contract,
its graph capture, the conditioned sampler loop without host synchronisation, and image-to-video on STDiT3 (XS/2 against
the oracle loop; XL/2 at the benchmark latent)."""
import pytest
import torch

from tests.models import stdit3_inputs, stdit3_pair
from tests.sampling_toys import toy_model
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _restated(vc, vu, z, fm, tc, tn, g, noise, update, N=1000):
    """fp32 contract of include/osb200.h osb_rf_masked_step -> (result fp32, changed-frame mask [B, T])."""
    fr = lambda m: m[:, None, :, None, None]  # noqa: E731
    ps = lambda v: v[:, None, None, None, None]  # noqa: E731
    m = fm * N
    x = z.float()
    changed = torch.zeros_like(fm, dtype=torch.bool)
    if update:
        upd = m >= tc[:, None]
        x = torch.where(fr(upd), x + ps((tc - tn) * (1.0 / N)) * (vu.float() + g * (vc.float() - vu.float())), x)
        prev, changed = upd, upd
    else:
        prev = fm == 1
    if noise is not None:
        add = (m >= tn[:, None]) & ~prev
        a = ps(tn * (1.0 / N))
        x = torch.where(fr(add), (1 - a) * x + a * noise.float(), x)
        changed = changed | add
    return x, changed


@pytest.mark.parametrize("shape", [(3, 4, 6, 8, 10), (3, 4, 5, 5, 7)])       # H*W % 8 == 0 (vector path) and not
@pytest.mark.parametrize("mode", ["fused", "update", "prologue"])
@pytest.mark.parametrize("in_place", [False, True])
def test_masked_step_kernel(shape, mode, in_place):
    _need_cuda()
    import osb200

    g = torch.Generator(device="cuda").manual_seed(7)
    B, C, T, H, W = shape
    vc, vu, z, noise = (torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4))
    fm = torch.tensor([[0.0, 0.5, 1.0, 0.25, 0.75, 1.0][:T], [1.0, 0.3, 0.0, 0.6, 0.5, 0.9][:T],
                       [0.5, 0.5, 1.0, 0.0, 0.45, 0.55][:T]], device="cuda")
    tc = torch.tensor([750.0, 600.0, 500.0], device="cuda")                      # per-sample schedules
    tn = torch.tensor([500.0, 300.0, 450.0], device="cuda")
    if mode == "prologue":
        tc = tn = torch.tensor([1000.0, 300.0, 500.0], device="cuda")
    update, nz = mode != "prologue", (noise if mode != "update" else None)
    ref, changed = _restated(vc, vu, z, fm, tc, tn, 6.5, nz, update)
    assert changed.any() and not changed.all()
    z_in = z.clone()
    out = osb200.rf_masked_step(vc if update else None, vu if update else None, z_in, fm, tc, tn, guidance=6.5, noise=nz,
                                update=update, out=z_in if in_place else None)
    torch.cuda.synchronize()
    assert (out.data_ptr() == z_in.data_ptr()) == in_place
    if not in_place:
        assert torch.equal(z_in, z)
    sel = changed[:, None, :, None, None].expand(shape)
    r, _ = report(f"rf_masked_step {mode} {shape} in_place={in_place}", out.float()[sel], ref[sel])
    assert r <= 2e-3
    assert torch.equal(out[~sel], z[~sel])                                        # frames left alone: bit for bit


def test_all_ones_mask_is_cfg_euler_bit_for_bit():
    _need_cuda()
    import osb200

    g = torch.Generator(device="cuda").manual_seed(3)
    shape = (2, 4, 16, 32, 32)
    vc, vu, z = (torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3))
    tc, tn = torch.full((2,), 733.0, device="cuda"), torch.full((2,), 466.5, device="cuda")
    dt = float(((tc - tn) / 1000)[0])
    a = osb200.cfg_euler(vc, vu, None, z, g_txt=7.0, dt=dt)
    b = osb200.rf_masked_step(vc, vu, z, torch.ones(2, 16, device="cuda"), tc, tn, guidance=7.0)
    assert torch.equal(a, b)


def test_all_ones_mask_sampler_is_the_t2v_loop():
    """RFLOW.sample with an all-ones frame mask (strategy [None]) returns the text-to-video loop's latent bit for bit."""
    _need_cuda()
    from opensora.schedulers import RFLOW

    g = torch.Generator(device="cuda").manual_seed(2)
    z = torch.randn(2, 4, 6, 8, 8, device="cuda", generator=g).to(torch.bfloat16)
    y = torch.randn(2, 1, 5, 8, device="cuda", generator=g)
    for transform in (False, True):
        sch = RFLOW(num_sampling_steps=7, cfg_scale=6.0, use_timestep_transform=transform)
        extra = dict(height=torch.full((2,), 360.0, device="cuda"), width=torch.full((2,), 640.0, device="cuda"),
                     num_frames=torch.full((2,), 51, device="cuda"))
        a = sch.sample(toy_model, z, y, y, additional_args=extra)
        b = sch.sample(toy_model, z, y, y, additional_args=extra, frame_mask=torch.ones(2, 6, device="cuda"))
        assert torch.equal(a, b), transform


def test_masked_step_graph_replay_reads_the_schedule():
    _need_cuda()
    import osb200

    g = torch.Generator(device="cuda").manual_seed(5)
    shape = (2, 4, 8, 16, 16)
    vc, vu, z, noise = (torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4))
    fm = torch.tensor([[0.0, 0.2, 0.4, 0.5, 0.6, 0.8, 1.0, 1.0]] * 2, device="cuda")
    tc, tn = torch.tensor([1000.0, 900.0], device="cuda"), torch.tensor([750.0, 700.0], device="cuda")
    out = torch.empty_like(z)
    osb200.rf_masked_step(vc, vu, z, fm, tc, tn, guidance=5.0, noise=noise, out=out)   # warm up outside the capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        osb200.rf_masked_step(vc, vu, z, fm, tc, tn, guidance=5.0, noise=noise, out=out)
    torch.cuda.current_stream().wait_stream(s)
    for a, b in (([500.0, 450.0], [250.0, 300.0]), ([600.0, 1000.0], [550.0, 450.0])):
        tc.copy_(torch.tensor(a))
        tn.copy_(torch.tensor(b))
        graph.replay()
        eager = osb200.rf_masked_step(vc, vu, z, fm, tc, tn, guidance=5.0, noise=noise)
        torch.cuda.synchronize()
        assert torch.equal(out, eager)


def test_conditioned_loop_never_synchronises():
    _need_cuda()
    from opensora.schedulers import RFLOW

    g = torch.Generator(device="cuda").manual_seed(1)
    B, C, T, H, W = 2, 4, 6, 8, 8
    z = torch.randn(B, C, T, H, W, device="cuda", generator=g).to(torch.bfloat16)
    y = torch.randn(B, 1, 5, 8, device="cuda", generator=g)
    fm = torch.tensor([[0.0, 0.5, 1.0, 1.0, 0.3, 1.0], [1.0, 1.0, 0.0, 0.7, 1.0, 1.0]], device="cuda")
    sch = RFLOW(num_sampling_steps=5, cfg_scale=6.0)
    sch.sample(toy_model, z, y, y, frame_mask=fm, generator=g)                   # warm up (module loads, caching allocator)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = sch.sample(toy_model, z, y, y, frame_mask=fm, generator=g)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(out[0, :, 0], z[0, :, 0]) and torch.equal(out[1, :, 2], z[1, :, 2])


def _i2v(cfg_name, B, T, H, W, steps, seed=11):
    """Strategy "0" (the first latent frame is the reference) through apply_mask_strategy and RFLOW.sample."""
    from opensora.schedulers import RFLOW
    from opensora.utils.inference_utils import apply_mask_strategy

    prod, oracle, cfg = stdit3_pair(cfg_name)
    inp = stdit3_inputs(cfg, B, T, H, W, lens=[cfg.model_max_length] + [17] * (B - 1), device="cuda")
    refs = [[torch.randn(cfg.in_channels, 2, H, W, generator=torch.Generator().manual_seed(seed + b)).cuda()] for b in range(B)]
    z = inp["x"].to(torch.bfloat16)
    fm = apply_mask_strategy(z, refs, ["0"] * B, loop_i=0)
    y_null = prod.y_embedder.y_embedding.detach()[None, None].repeat(B, 1, 1, 1)
    extra = dict(fps=inp["fps"], height=inp["height"], width=inp["width"])
    with torch.no_grad():
        out = RFLOW(num_sampling_steps=steps, cfg_scale=4.0).sample(prod, z, inp["y"], y_null, mask=inp["mask"],
                                                                    additional_args=extra, frame_mask=fm,
                                                                    generator=torch.Generator(device="cuda").manual_seed(seed))
    return out, z, fm, refs, (oracle, inp, y_null, extra)


def test_xs_image_to_video_vs_oracle_loop():
    _need_cuda()
    from tests import rf_conditioning_ref as R

    steps = 4
    out, z, fm, refs, (oracle, inp, y_null, extra) = _i2v("xs", 2, 6, 8, 8, steps)
    assert torch.equal(fm.cpu(), torch.tensor([[0.0] + [1.0] * 5] * 2))
    g = torch.Generator(device="cuda").manual_seed(11)
    ns = [torch.randn(z.shape, generator=g, device="cuda", dtype=torch.bfloat16).float() for _ in range(steps)]
    oracle = oracle.cuda()
    with torch.no_grad():
        ref = R.rflow_sample_masked(lambda x, t, y, **kw: oracle(x, t, y, **kw), z.float(), inp["y"], y_null.float(), fm, ns,
                                    mask=inp["mask"], steps=steps, cfg_scale=4.0, **extra)
        ob = oracle.to(torch.bfloat16)
        noise = R.rflow_sample_masked(lambda x, t, y, **kw: ob(x.to(torch.bfloat16).float(), t, y, **kw).float(), z.float(),
                                      inp["y"], y_null.float(), fm, ns, mask=inp["mask"], steps=steps, cfg_scale=4.0, **extra)
    r, _ = report("STDiT3-XS/2 i2v 4 steps vs oracle loop", out, ref)
    rn = rel_l2(noise, ref)
    print(f"[parity] oracle-loop-in-bf16 noise floor rel_l2={rn:.3e}")
    assert r < max(1.5 * rn, 1e-2) and r < 6e-2, (r, rn)
    for b in range(2):
        assert torch.equal(out[b, :, 0], refs[b][0][:, 0].to(torch.bfloat16))    # the image, bit for bit


def test_xl_image_to_video_at_the_benchmark_latent():
    _need_cuda()
    out, z, fm, refs, _ = _i2v("xl", 1, 64, 32, 32, 3)
    assert torch.isfinite(out).all()
    assert torch.equal(out[0, :, 0], refs[0][0][:, 0].to(torch.bfloat16))
    assert not torch.equal(out[0, :, 1:], z[0, :, 1:])
