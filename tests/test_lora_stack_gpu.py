"""Several LoRA / DoRA adapters at once on MMDiT on the GPU: the small-config model with a LoRA, DoRA, LoRA stack on every
block Linear, on the bf16 GEMMs and on the FP8 GEMMs (`enable_fp8(projections=True, lora=True)`), against the fp32
oracle on the weights merged by peft's recursion (tests/test_lora_stack_cpu.py); and a stack of one adapter, bit for bit
and launch for launch the forward of that adapter alone."""
import pytest
import torch

from tests import mmdit_fp8_lora_ref as LR
from tests import mmdit_fp8_proj_ref as PR
from tests import mmdit_fp8_ref as MR
from tests.adapters import load_stack, stack_registry, stacked_state, write_stack
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu

NAMES, WEIGHTS = ["a", "b", "c"], (1.0, 0.8, 1.25)


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _block_linears(m):
    return m.fp8_mlp_linears() + m.fp8_proj_linears()


def _oracle(W32, cfg, inp):
    from oracle import mmdit_oracle as M

    f = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    return M.model_forward(W32, cfg, f["img"], f["img_ids"], f["txt"], f["txt_ids"], f["timesteps"], f["y_vec"],
                           cond=f["cond"], guidance=f["guidance"])


def _small(fused, liger):
    m = mmdit_model(fused, liger).cuda()
    inp = {k: v.cuda() for k, v in mmdit_inputs(2, 40, (3, 6, 8), guidance=[4.0, 7.5]).items()}
    return m, dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger), inp


@pytest.mark.parametrize("fused,liger", [(True, False), (False, True)])
def test_small_mmdit_bf16_stack_against_the_oracle(tmp_path, fused, liger):
    """tests/test_dora_gpu.py's bars: within 1e-2 of the fp32 oracle on the merged weights and within 1.1x the error of
    the same model without adapters against its own oracle."""
    m, cfg, inp = _small(fused, liger)
    with torch.no_grad():
        base = m(**inp)
        base_err = rel_l2(base, _oracle({k: v.float() for k, v in m.state_dict().items()}, cfg, inp))
        load_stack(m, write_stack(tmp_path, m, ("lora", "dora", "lora"), targets=_block_linears(m), rel=0.3), NAMES,
                   WEIGHTS)
        out = m(**inp)
    r, _ = report(f"MMDiT + LoRA, DoRA, LoRA stack fused_qkv={fused} liger={liger}", out, _oracle(
        stacked_state(m, NAMES, WEIGHTS), cfg, inp))
    print(f"[parity] same model without adapters vs its fp32 oracle: rel_l2={base_err:.3e}")
    assert rel_l2(out, base) > 5 * r, "the stack must change the output well above the error"
    assert r <= 1e-2 and r <= 1.1 * base_err, (r, base_err)


@pytest.mark.parametrize("fused,liger,attn", [(True, False, False), (False, True, True)])
def test_small_mmdit_fp8_stack_against_the_oracle(tmp_path, fused, liger, attn):
    """tests/test_mmdit_fp8_lora_gpu.py's bars: within 1.1x the error of the FP8 emulation with the stack, and 1e-2."""
    m, cfg, inp = _small(fused, liger)
    load_stack(m, write_stack(tmp_path, m, ("lora", "dora", "lora"), targets=_block_linears(m), rel=0.3, r=64),
               NAMES, WEIGHTS)
    m.enable_fp8(projections=True, lora=True)
    if attn:
        m.enable_fp8_attention()
    with torch.no_grad():
        out = m(**inp)
    ref = _oracle(stacked_state(m, NAMES, WEIGHTS), cfg, inp)
    rows, ads = stack_registry(m)
    saved = MR._lin
    MR._lin = LR._lin_with(rows, ads, saved)
    try:
        from oracle import mmdit_oracle as M
        from tests import mmdit_fp8_attn_ref as AR

        with PR.fp8_projections(), (AR.fp8_attention() if attn else torch.no_grad()):
            emu = M.model_forward(LR.emulation_state(m), cfg, inp["img"], inp["img_ids"], inp["txt"], inp["txt_ids"],
                                  inp["timesteps"].to(torch.bfloat16), inp["y_vec"], cond=inp["cond"],
                                  guidance=inp["guidance"].to(torch.bfloat16))
    finally:
        MR._lin = saved
    r, _ = report(f"MMDiT C=256 FP8 + LoRA, DoRA, LoRA stack fused={fused} liger={liger} attn={attn}", out, ref)
    r_emu = rel_l2(emu, ref)
    print(f"[mmdit fp8 lora stack] emulation rel_l2={r_emu:.3e}, ratio {r / r_emu:.3f}")
    assert r <= 1.1 * r_emu and r < 1e-2, (r, r_emu)


def test_one_adapter_stack_is_the_single_adapter_forward(tmp_path):
    """The bits and launch count of a model holding one DoRA adapter, against: the same adapter made the only active
    one of a two-adapter model (`set_adapters`), and the same adapter left after `unload_lora` of the other."""
    import osb200

    from opensora.utils.lora import load_lora, set_adapters, unload_lora

    def run(m):
        with torch.no_grad():
            m(**inp)
            n0 = osb200.launch_count()
            out = m(**inp)
            return out, osb200.launch_count() - n0

    m1, cfg, inp = _small(True, False)
    p_d, p_l = write_stack(tmp_path, m1, ("dora", "lora"), targets=_block_linears(m1) + ["img_in", "txt_in"])
    want = run(load_lora(m1, p_d))
    m2 = _small(True, False)[0]
    load_stack(m2, [p_l, p_d], ["l", "d"])
    both = run(m2)
    set_adapters(m2, ["d"])
    got = run(m2)
    m3 = _small(True, False)[0]
    load_stack(m3, [p_d, p_l], ["d", "l"])
    unload_lora(m3, "l")
    got3 = run(m3)
    assert not torch.equal(both[0], want[0])
    for out, n in (got, got3):
        assert torch.equal(out, want[0]) and n == want[1], (n, want[1])
