"""GPU parity of the osb200 MMDiT block processors / model (through the C ABI) against `oracle/mmdit_oracle.py`,
which tests/test_oracle_cpu.py pins to fixtures produced by executing the reference's own source
(opensora/models/mmdit/{layers,math,model}.py).  Identical bf16-rounded weights and inputs on both sides."""
import pytest
import torch

from tests.models import MMDIT_CFG, mmdit_ids, mmdit_model
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fused,liger,thw", [(True, False, (3, 6, 8)), (False, False, (3, 6, 8)), (False, True, (3, 6, 8)),
                                              (False, True, (5, 12, 16))])
def test_mmdit_model_vs_pinned_oracle(fused, liger, thw):
    """(False, True) = the layout the reference ships (configs/diffusion/inference/256px.py:40-41); the last case has a
    1000-token joint sequence (streaming attention, 8 key blocks)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import mmdit_oracle as M

    m = mmdit_model(fused, liger, device="cuda")
    B, Lt = 2, 40
    T, H, W = thw
    g = torch.Generator().manual_seed(3)
    rb = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)  # noqa: E731
    txt_ids, img_ids = mmdit_ids(B, Lt, T, H, W)
    inp = dict(img=rb(B, T * H * W, 64), img_ids=img_ids, txt=rb(B, Lt, 128), txt_ids=txt_ids,
               timesteps=torch.tensor([0.3, 0.8]), y_vec=rb(B, 96), cond=rb(B, T * H * W, 68), guidance=torch.tensor([4.0, 7.5]))
    with torch.no_grad():
        out = m(**{k: v.cuda() for k, v in inp.items()})
    W32 = {k: v.float() for k, v in m.state_dict().items()}
    cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
    finp = {k: (v.float() if v.is_floating_point() else v).cuda() for k, v in inp.items()}
    ref = M.model_forward(W32, cfg, finp["img"], finp["img_ids"], finp["txt"], finp["txt_ids"], finp["timesteps"],
                          finp["y_vec"], cond=finp["cond"], guidance=finp["guidance"])
    Wb = {k: v for k, v in m.state_dict().items()}
    binp = {k: v.cuda() for k, v in inp.items()}
    noise = M.model_forward(Wb, cfg, binp["img"], binp["img_ids"], binp["txt"], binp["txt_ids"], binp["timesteps"].to(torch.bfloat16),
                            binp["y_vec"], cond=binp["cond"], guidance=binp["guidance"].to(torch.bfloat16))
    r, _ = report(f"MMDiT model fused_qkv={fused} liger={liger} L={Lt + T * H * W}", out, ref)
    rn = rel_l2(noise, ref)
    print(f"[parity] reference-in-bf16 noise floor rel_l2={rn:.3e}")
    assert out.shape == ref.shape
    # the bar sits well below the reference-in-bf16 floor, not at it
    assert r < 1.0e-2 and r < rn


def test_processor_hook_is_the_plugin_point():
    """`block.set_processor(p)` (layers.py:299-300) swaps the implementation: a wrapping processor sees the calls."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from opensora.models.mmdit.layers import DoubleStreamBlockProcessor

    m = mmdit_model(True, device="cuda")
    calls = []

    class Spy(DoubleStreamBlockProcessor):
        def __call__(self, attn, img, txt, vec, pe):
            calls.append(img.shape)
            return super().__call__(attn, img, txt, vec, pe)

    for b in m.double_blocks:
        assert isinstance(b.get_processor(), DoubleStreamBlockProcessor)
        b.set_processor(Spy())
    txt_ids, img_ids = mmdit_ids(1, 8, 1, 4, 4)
    with torch.no_grad():
        out = m(img=torch.randn(1, 16, 64).cuda(), img_ids=img_ids.cuda(), txt=torch.randn(1, 8, 128).cuda(), txt_ids=txt_ids.cuda(),
                timesteps=torch.tensor([0.5]).cuda(), y_vec=torch.randn(1, 96).cuda(), cond=torch.randn(1, 16, 68).cuda(),
                guidance=torch.tensor([4.0]).cuda())
    assert len(calls) == 2 and out.shape == (1, 16, 64) and torch.isfinite(out).all()
