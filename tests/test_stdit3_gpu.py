"""End-to-end parity of the osb200 STDiT3 against the fp32 oracle holding identical bf16-rounded
weights, on identical seeded latents / timesteps / text embeddings.

Tolerance (north_star: 'within 1e-3 rel of the reference', made meaningful for bf16 in SURVEY.md §7
hard part 2): the product rounds the residual stream and every GEMM output to bf16 exactly where the
reference's own bf16 path does, so its error vs the fp32 oracle must not exceed the error of the
oracle itself run in bf16 (the reference-precision noise floor, measured in the same test) by more
than 1.1x, and must stay below an absolute
1.5e-2 (depth 2) / 3e-2 (depth 28) rel-L2."""
import pytest
import torch

from tests.models import stdit3_pair
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu


def _run(cfg_name, B, T, H, W, x_mask=None, lens=None):
    from oracle import stdit3_oracle as O

    prod, oracle, cfg = stdit3_pair(cfg_name)
    inp = O.synthetic_inputs(cfg, B=B, T=T, H=H, W=W, lens=lens)
    inp = {k: (v.to(torch.bfloat16).float() if v.is_floating_point() else v).cuda() for k, v in inp.items()}
    if x_mask is not None:
        inp["x_mask"] = x_mask.cuda()
    oracle = oracle.cuda()
    with torch.no_grad():
        ref = oracle(**inp)
        out = prod(**inp)
        noise = oracle.to(torch.bfloat16)(**inp)   # the oracle at the reference's own precision
    return out, ref, noise


@pytest.mark.parametrize("B,T,H,W", [(1, 8, 16, 16), (2, 4, 8, 12)])
def test_xs_parity(B, T, H, W):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out, ref, noise = _run("xs", B, T, H, W)
    r, _ = report(f"STDiT3-XS/2 B{B} {T}x{H}x{W}", out, ref)
    rn = rel_l2(noise, ref)
    print(f"[parity] oracle-in-bf16 noise floor rel_l2={rn:.3e}")
    assert out.shape == ref.shape
    assert r < 1.5e-2 and r < 1.1 * rn


def test_xs_x_mask_and_ragged_text():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    xm = torch.ones(2, 6, dtype=torch.bool)
    xm[0, 0] = False
    xm[1, 2:4] = False
    out, ref, noise = _run("xs", 2, 6, 8, 8, x_mask=xm, lens=[300, 17])
    r, _ = report("STDiT3-XS/2 x_mask", out, ref)
    rn = rel_l2(noise, ref)
    assert r < 1.5e-2 and r < 1.1 * rn


def test_xl_parity_reduced_latent():
    """Full-depth STDiT3-XL/2 (28x2 blocks, C=1152, 16 heads x 72) on a 16x16x16 latent."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out, ref, noise = _run("xl", 1, 16, 16, 16)
    r, _ = report("STDiT3-XL/2 16x16x16", out, ref)
    rn = rel_l2(noise, ref)
    print(f"[parity] oracle-in-bf16 noise floor rel_l2={rn:.3e}")
    assert r < 3e-2 and r < 1.1 * rn   # measured 2.15e-2 against a floor of 2.22e-2


def _block_trace(prod, oracle, inp):
    """Residual stream after every block of the product (bf16) and of the fp32 oracle: SURVEY.md 8d "Parity report"
    (first-divergence localisation)."""
    ref_x, got_x = [], []
    hooks = [b.register_forward_hook(lambda m, a, out: ref_x.append(out.detach().float()))
             for pair in zip(oracle.spatial_blocks, oracle.temporal_blocks) for b in pair]
    orig = prod._block

    def traced(osb, blk, bi, xs, *a, **k):
        r = orig(osb, blk, bi, xs, *a, **k)
        got_x.append(xs.detach().float().clone())
        return r

    prod._block = traced
    try:
        with torch.no_grad():
            ref = oracle(**inp)
            out = prod(**inp)
    finally:
        prod._block = orig
        for h in hooks:
            h.remove()
    per_block = [rel_l2(g.view_as(r), r) for g, r in zip(got_x, ref_x)]
    return out, ref, per_block


def test_xl_parity_at_the_benchmark_shape():
    """STDiT3-XL/2, full depth, on the BASELINE.json latent 1x4x64x32x32 (T = 64, S = 256, 16 384 tokens: two query tiles
    per spatial sequence, two temporal sequences packed per tile, 3 text key tiles) against the fp32 oracle on the same GPU,
    with the per-block error trace.  Bars: final output within 1.5x of the oracle's own bf16 noise floor (measured here) and
    below 3e-2; the residual stream may not jump by more than 3x between consecutive blocks (a broken block would)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import stdit3_oracle as O

    prod, oracle, cfg = stdit3_pair("xl")
    inp = O.synthetic_inputs(cfg, B=1, T=64, H=32, W=32, lens=[260])
    inp = {k: (v.to(torch.bfloat16).float() if v.is_floating_point() else v).cuda() for k, v in inp.items()}
    oracle = oracle.cuda()
    out, ref, per_block = _block_trace(prod, oracle, inp)
    with torch.no_grad():
        noise = oracle.to(torch.bfloat16)(**inp)
    r, _ = report("STDiT3-XL/2 64x32x32 (benchmark shape)", out, ref)
    rn = rel_l2(noise, ref)
    print(f"[parity] oracle-in-bf16 noise floor rel_l2={rn:.3e}")
    print("[parity] residual stream rel_l2 after block k: " + " ".join(f"{k}:{e:.1e}" for k, e in enumerate(per_block)))
    assert len(per_block) == 2 * cfg.depth
    assert torch.isfinite(out).all()
    assert per_block[0] < 5e-3, per_block[0]
    for k in range(1, len(per_block)):
        assert per_block[k] < 3.0 * per_block[k - 1] + 2e-3, (k, per_block[k - 1], per_block[k])
    assert r < 3e-2 and r < 1.1 * rn, (r, rn)   # measured 2.16e-2 against a floor of 2.23e-2

