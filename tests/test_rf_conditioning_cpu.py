"""Image / video conditioning of STDiT3's sampler on the CPU: the mask-strategy helpers of
`opensora.utils.inference_utils` on hand-computed cases, the properties of the fp32 oracle loop
(`tests/rf_conditioning_ref.py::rflow_sample_masked`), and `RFLOW.sample(frame_mask=...)` through the CPU stand-in of
the binding around a toy model and around the real host-side STDiT3 against the oracle loop.  Like the v1.2 sampler itself
this path is restated, not pinned by the reference.  The kernel is checked on the GPU (test_rf_conditioning_gpu)."""
import pytest
import torch

from tests import rf_conditioning_ref as R
from tests.models import stdit3_pair
from tests.util import rel_l2


def _toy(x, timestep, y, mask=None, fps=None, x_mask=None, **kw):
    """[2B, C, T, H, W] -> [2B, 2C, T, H, W] fp32 (velocity | sigma halves); ignores x_mask."""
    f = x.float()
    cap = y.float().mean(dim=(1, 2, 3))[:, None, None, None, None]
    v = torch.tanh(0.8 * f + cap) * (0.5 + timestep.float()[:, None, None, None, None] / 1000.0)
    return torch.cat((v, 0.1 * f), dim=1)


def _noises(shape, steps, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(shape, generator=g, dtype=dtype) for _ in range(steps)]


# ---- mask strategy helpers ------------------------------------------------------------------------------------------
def test_parse_mask_strategy_and_nearest_point():
    from opensora.utils.inference_utils import find_nearest_point, parse_mask_strategy

    assert parse_mask_strategy(None) == [] and parse_mask_strategy("") == []
    assert parse_mask_strategy("0") == [[0, 0, 0, 0, 1, 0.0]]
    assert parse_mask_strategy("0,1,2") == [[0, 1, 2, 0, 1, 0.0]]
    got = parse_mask_strategy("0,0,0,0,8,0.3;1,2,-3,4,5,0.5")
    assert got == [[0, 0, 0, 0, 8, 0.3], [1, 2, -3, 4, 5, 0.5]]
    assert all(type(v) is int for v in got[1][:5]) and type(got[1][5]) is float
    with pytest.raises(ValueError):
        parse_mask_strategy("0,0,0,0,1,0,7")
    # t = value // point, one up when past the half way and t < max_value // point - 1
    assert find_nearest_point(7, 5, 20) == 5       # 7 % 5 = 2 <= 2.5: down
    assert find_nearest_point(8, 5, 20) == 10      # 3 > 2.5 and 1 < 3: up
    assert find_nearest_point(18, 5, 20) == 15     # 3 > 2.5 but 3 == 20 // 5 - 1: down
    assert find_nearest_point(10, 5, 20) == 10


def test_apply_mask_strategy_hand_computed():
    from opensora.utils.inference_utils import apply_mask_strategy

    C, T, H, W = 2, 10, 1, 1
    ref = torch.arange(1, 1 + C * 6, dtype=torch.float32).view(C, 6, H, W)          # [C, 6, H, W], frame values distinct
    z = torch.zeros(3, C, T, H, W)
    m = apply_mask_strategy(z, [[ref], [ref], None], ["0", "0,0,-2,-3,5,0.5", None], loop_i=0)
    assert m.dtype == torch.float32 and m.shape == (3, T)
    # "0" = 0,0,0,0,1,0: reference frame 0 at frame 0, kept
    assert torch.equal(m[0], torch.tensor([0.0] + [1.0] * 9))
    assert torch.equal(z[0, :, 0], ref[:, 0]) and not z[0, :, 1:].any()
    # negative starts from the end (ref 6 - 2 = 4, target 10 - 3 = 7); length 5 clipped to min(10 - 7, 6 - 4) = 2
    assert torch.equal(m[1], torch.tensor([1.0] * 7 + [0.5, 0.5, 1.0]))
    assert torch.equal(z[1, :, 7:9], ref[:, 4:6]) and not z[1, :, :7].any() and not z[1, :, 9:].any()
    assert torch.equal(m[2], torch.ones(T)) and not z[2].any()                      # None: nothing applies
    # loop_id filtering: entries of loop 1 do nothing in loop 0
    z = torch.zeros(1, C, T, H, W)
    assert torch.equal(apply_mask_strategy(z, [[ref]], ["1,0,0,0,3,0"], loop_i=0), torch.ones(1, T)) and not z.any()
    m = apply_mask_strategy(z, [[ref]], ["1,0,0,0,3,0"], loop_i=1)
    assert torch.equal(m[0, :4], torch.tensor([0.0, 0.0, 0.0, 1.0])) and torch.equal(z[0, :, :3], ref[:, :3])
    # [None] -> an all-ones mask; [] -> None
    assert torch.equal(apply_mask_strategy(torch.zeros(1, C, T, H, W), [None], [None], 0), torch.ones(1, T))
    assert apply_mask_strategy(torch.zeros(1, C, T, H, W), [], [], 0) is None


def test_apply_mask_strategy_align_snaps_both_branches():
    from opensora.utils.inference_utils import apply_mask_strategy

    C, T = 1, 20
    ref = torch.arange(12, dtype=torch.float32).view(C, 12, 1, 1) + 100
    z = torch.zeros(2, C, T, 1, 1)
    # sample 0: ref_start 3 -> 5 (3 % 5 > 2.5, 0 < 12 // 5 - 1), target 8 -> 10 (1 < 20 // 5 - 1); length 4
    # sample 1: ref_start 2 -> 0 (2 % 5 <= 2.5), target 13 -> 15 (3 > 2.5, 2 < 3) ; target 18 would stay 15 (3 == 3)
    m = apply_mask_strategy(z, [[ref], [ref]], ["0,0,3,8,4,0", "0,0,2,13,3,0.25"], loop_i=0, align=5)
    assert torch.equal(z[0, 0, 10:14, 0, 0], ref[0, 5:9, 0, 0]) and torch.equal(m[0, 10:14], torch.zeros(4))
    assert float(m[0].sum()) == T - 4
    assert torch.equal(z[1, 0, 15:18, 0, 0], ref[0, 0:3, 0, 0]) and torch.equal(m[1, 15:18], torch.full((3,), 0.25))
    z = torch.zeros(1, C, T, 1, 1)
    m = apply_mask_strategy(z, [[ref]], ["0,0,0,18,9,0"], loop_i=0, align=5)       # 18 -> 15 (upper bound), length 5
    assert torch.equal(m[0, 15:], torch.zeros(5)) and torch.equal(z[0, 0, 15:, 0, 0], ref[0, 0:5, 0, 0])


def test_append_generated_adds_reference_and_entry():
    from opensora.utils.inference_utils import append_generated

    gen = torch.randn(2, 4, 8, 2, 2)
    refs, ms = append_generated(None, gen, [None, [torch.zeros(4, 3, 2, 2)]], ["", "0"], 1, 3, 0.2, is_latent=True)
    assert len(refs[0]) == 1 and torch.equal(refs[0][0], gen[0])
    assert len(refs[1]) == 2 and torch.equal(refs[1][1], gen[1])
    assert ms == ["1,0,-3,0,3,0.2", "0;1,1,-3,0,3,0.2"]

    class _Enc:
        def encode(self, x):
            return x * 2

    refs, _ = append_generated(_Enc(), gen, [None, None], [None, None], 1, 3, 0.0)
    assert torch.equal(refs[0][0], gen[0] * 2)


# ---- the oracle loop ------------------------------------------------------------------------------------------------
def _oracle_inputs(B=2, C=3, T=4, H=4, W=6, L=5, seed=3):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, C, T, H, W, generator=g).to(torch.bfloat16).float()
    y, y_null = torch.randn(B, 1, L, 8, generator=g), torch.randn(B, 1, L, 8, generator=g)
    return z, y, y_null


def test_oracle_all_ones_mask_is_the_t2v_loop():
    from oracle import sampling_oracle as O

    z, y, y_null = _oracle_inputs()
    ns = [n.float() for n in _noises(z.shape, 5, 1)]
    ref = O.rflow_sample(_toy, z, y, y_null, steps=5, cfg_scale=6.0)
    out = R.rflow_sample_masked(_toy, z, y, y_null, torch.ones(2, 4), ns, steps=5, cfg_scale=6.0)
    assert torch.equal(out, ref)


def test_oracle_kept_and_edited_frames():
    """mask [0, 0.5, 1, 1], 4 steps (t = 1000, 750, 500, 250): frame 0 never changes; frame 1 is the reference at t = 1000
    and 750, is re-noised at t = 500 to (1 - 0.5) x0 + 0.5 noise_2 and generated after; only noise_2 reaches the output."""
    z, y, y_null = _oracle_inputs()
    fm = torch.tensor([[0.0, 0.5, 1.0, 1.0]] * 2)
    ns = [n.float() for n in _noises(z.shape, 4, 2)]
    seen = []

    def spy(x, t, y, **kw):
        seen.append((x[: x.shape[0] // 2].clone(), float(t[0]), kw["x_mask"].clone()))
        return _toy(x, t, y, **kw)

    out = R.rflow_sample_masked(spy, z, y, y_null, fm, ns, steps=4, cfg_scale=5.0)
    assert torch.equal(out[:, :, 0], z[:, :, 0])
    assert [s[1] for s in seen] == [1000.0, 750.0, 500.0, 250.0]
    for i, (x, t, xm) in enumerate(seen):
        assert torch.equal(xm, (fm * 1000 >= t).repeat(2, 1))
        assert torch.equal(x[:, :, 0], z[:, :, 0])
        if t > 500:
            assert torch.equal(x[:, :, 1], z[:, :, 1])
    assert torch.equal(seen[2][0][:, :, 1], 0.5 * z[:, :, 1] + 0.5 * ns[2][:, :, 1])
    assert not torch.equal(seen[3][0][:, :, 1], seen[2][0][:, :, 1])              # generated from t = 500 on
    # re-noised once: the other steps' noise reaches no frame (mask-1 frames start from z itself)
    other = [n if i == 2 else torch.randn_like(n) for i, n in enumerate(ns)]
    assert torch.equal(R.rflow_sample_masked(_toy, z, y, y_null, fm, other, steps=4, cfg_scale=5.0), out)


# ---- the sampler through the binding stand-in ------------------------------------------------------------------------
def test_sampler_masked_loop_vs_oracle_toy(fake_osb):
    from opensora.schedulers import RFLOW

    z, y, y_null = _oracle_inputs(B=3)
    fm = torch.tensor([[0.0, 0.5, 1.0, 1.0], [1.0, 0.3, 0.0, 0.75], [1.0, 1.0, 1.0, 1.0]])
    z0 = z.to(torch.bfloat16)
    out = RFLOW(num_sampling_steps=6, cfg_scale=5.0).sample(_toy, z0, y, y_null, frame_mask=fm,
                                                            generator=torch.Generator().manual_seed(11))
    ref = R.rflow_sample_masked(_toy, z, y, y_null, fm, [n.float() for n in _noises(z.shape, 6, 11)], steps=6, cfg_scale=5.0)
    assert out.dtype == torch.bfloat16 and rel_l2(out, ref) < 2e-2
    assert torch.equal(out[0, :, 0], z0[0, :, 0]) and torch.equal(out[1, :, 2], z0[1, :, 2])
    names = [c[0] for c in fake_osb.calls]
    assert names.count("rf_masked_step") == 1 + 6 and "cfg_euler" not in names


def test_sampler_without_frame_mask_is_unchanged(fake_osb):
    """frame_mask=None keeps the text-to-video loop: one osb_cfg_euler per step, the same latent as that loop restated."""
    from opensora.schedulers import RFLOW

    z, y, y_null = _oracle_inputs()
    z0 = z.to(torch.bfloat16)
    out = RFLOW(num_sampling_steps=4, cfg_scale=5.0).sample(_toy, z0, y, y_null)
    calls = list(fake_osb.calls)
    fake_osb.reset()
    x = z0
    ts = [(1.0 - i / 4) * 1000.0 for i in range(4)] + [0.0]
    for i in range(4):
        t = torch.full((2,), ts[i])
        vc, vu = (p.to(torch.bfloat16) for p in _toy(torch.cat((x, x)), torch.cat((t, t)), torch.cat((y, y_null))).chunk(2, 1)[0].chunk(2))
        dt = (t - torch.full((2,), ts[i + 1])) / 1000
        x = fake_osb.cfg_euler(vc, vu, None, x, g_txt=5.0, dt=float(dt[0]))
    assert torch.equal(out, x)
    assert calls == fake_osb.calls


def test_sampler_all_ones_mask_matches_t2v(fake_osb):
    from opensora.schedulers import RFLOW

    z, y, y_null = _oracle_inputs()
    z0 = z.to(torch.bfloat16)
    a = RFLOW(num_sampling_steps=4, cfg_scale=5.0).sample(_toy, z0, y, y_null)
    b = RFLOW(num_sampling_steps=4, cfg_scale=5.0).sample(_toy, z0, y, y_null, frame_mask=torch.ones(2, 4))
    assert torch.equal(a, b)


def test_rflow_conditioned_sampler_drives_the_model(fake_osb):
    """RFLOW.sample(frame_mask=...) around the REAL host-side STDiT3 against the oracle loop around the fp32 oracle model,
    both fed the same per-step noise: 4 steps, frame masks [0, 0.5, 1, 1] and [1, 0, 0.5, 1]."""
    from oracle import stdit3_oracle as OS
    from opensora.schedulers import RFLOW

    prod, oracle, cfg = stdit3_pair("xs", device="cpu")
    B, steps = 2, 4
    inp = OS.synthetic_inputs(cfg, B=B, T=4, H=8, W=8, lens=[cfg.model_max_length, 11])
    inp = {k: (v.to(torch.bfloat16).float() if v.is_floating_point() else v) for k, v in inp.items()}
    y_null = prod.y_embedder.y_embedding.detach()[None, None].repeat(B, 1, 1, 1)
    extra = dict(fps=inp["fps"], height=inp["height"], width=inp["width"])
    fm = torch.tensor([[0.0, 0.5, 1.0, 1.0], [1.0, 0.0, 0.5, 1.0]])
    z0 = inp["x"].to(torch.bfloat16)
    seen = []

    def spy(x, t, y, **kw):
        seen.append(kw["x_mask"].clone())
        return prod(x, t, y, **kw)

    with torch.no_grad():
        out = RFLOW(num_sampling_steps=steps, cfg_scale=4.0).sample(spy, z0, inp["y"], y_null, mask=inp["mask"],
                                                                    additional_args=extra, frame_mask=fm,
                                                                    generator=torch.Generator().manual_seed(21))
        ns = [n.float() for n in _noises(z0.shape, steps, 21)]
        ref = R.rflow_sample_masked(lambda x, t, y, **kw: oracle(x, t, y, **kw), z0.float(), inp["y"], y_null.float(), fm, ns,
                                    mask=inp["mask"], steps=steps, cfg_scale=4.0, **extra)
        ob = oracle.to(torch.bfloat16)
        noise = R.rflow_sample_masked(lambda x, t, y, **kw: ob(x.to(torch.bfloat16).float(), t, y, **kw).float(), z0.float(),
                                      inp["y"], y_null.float(), fm, ns, mask=inp["mask"], steps=steps, cfg_scale=4.0, **extra)
    assert out.shape == z0.shape and out.dtype == torch.bfloat16
    r, rn = rel_l2(out, ref), rel_l2(noise, ref)
    assert r < max(1.5 * rn, 1e-2) and r < 6e-2, (r, rn)
    assert torch.equal(out[0, :, 0], z0[0, :, 0]) and torch.equal(out[1, :, 1], z0[1, :, 1])
    ts = [1000.0, 750.0, 500.0, 250.0]
    assert len(seen) == steps
    for xm, t in zip(seen, ts):
        assert xm.dtype == torch.bool and torch.equal(xm, (fm * 1000 >= t).repeat(2, 1))
    names = [c[0] for c in fake_osb.calls]
    assert names.count("rf_masked_step") == 1 + steps and "cfg_euler" not in names


def test_looped_driver_conditions_each_clip_on_the_last(fake_osb, monkeypatch):
    from opensora.schedulers import RFLOW
    from opensora.utils.inference_utils import sample_looped

    B, C, T, H, W, L = 1, 3, 8, 4, 4, 3
    _, y, y_null = _oracle_inputs(B=B)
    sch = RFLOW(num_sampling_steps=3, cfg_scale=5.0)
    clips, masks = [], []
    real = sch.sample

    def spy(model, z, y, y_null, frame_mask=None, **kw):
        masks.append(None if frame_mask is None else frame_mask.clone())
        clips.append(real(model, z, y, y_null, frame_mask=frame_mask, **kw))
        return clips[-1]

    monkeypatch.setattr(sch, "sample", spy)
    refs, ms = [None], [None]
    out = sample_looped(sch, _toy, (B, C, T, H, W), y, y_null, refs, ms, num_loop=2, condition_frame_length=L,
                        generator=torch.Generator().manual_seed(4))
    assert len(clips) == 2 and out.shape == (B, C, T + (T - L), H, W)
    assert torch.equal(masks[0], torch.ones(B, T))
    assert torch.equal(masks[1], torch.tensor([[0.0] * L + [1.0] * (T - L)]))
    assert torch.equal(clips[1][:, :, :L], clips[0][:, :, T - L:])                  # edit 0: kept bit for bit
    assert torch.equal(out[:, :, :T], clips[0]) and torch.equal(out[:, :, T:], clips[1][:, :, L:])
    assert ms == [f"1,0,-{L},0,{L},0.0"] and len(refs[0]) == 1
