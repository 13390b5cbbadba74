"""The FP8 (e4m3) projection path of MMDiT on the GPU: the block-scaled output mode of the FP8 attention kernel
(osb_attn_fp8_blocks) against the block rule and the same kernel's bf16 output, and the full-width model with every block
Linear on FP8 against the fp32 oracle, with the emulation reference of tests/mmdit_fp8_proj_ref.py as the yardstick."""
import contextlib

import pytest
import torch

from tests import mmdit_fp8_attn_ref as AR
from tests import mmdit_fp8_proj_ref as PR
from tests.models import MMDIT_CFG, MMDIT_WIDE, mmdit_inputs, mmdit_model
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


@pytest.mark.parametrize("L", [77, 1000, 2560, 8828])
def test_block_output_mode(L):
    """B = 3, H = 24, codes and scales written into column slices of [rows, 5C] / [rows, 5H] buffers."""
    import osb200

    B, H = 3, 24
    C = H * 128
    qkv, kw = AR.operands_cuda(B, L, H, True, min(256, L // 2))
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    ws = osb200.attn_fp8_workspace(B, L, H, "cuda")
    bf = torch.zeros(B * L, C, dtype=torch.bfloat16, device="cuda")
    osb200.attn_fp8(q, k, v, bf, workspace=ws, **kw)
    codes = torch.zeros(B * L, 5 * C, dtype=torch.float8_e4m3fn, device="cuda")
    scales = torch.full((B * L, 5 * H), -1.0, device="cuda")
    osb200.attn_fp8_blocks(q, k, v, codes[:, :C], scales[:, :H], workspace=ws, **kw)
    first = (codes.clone(), scales.clone())
    osb200.attn_fp8_blocks(q, k, v, codes[:, :C], scales[:, :H], workspace=ws, **kw)
    torch.cuda.synchronize()
    assert torch.equal(codes.view(torch.uint8), first[0].view(torch.uint8)) and torch.equal(scales, first[1])
    assert not codes[:, C:].view(torch.uint8).any() and torch.all(scales[:, H:] == -1.0)   # nothing outside the slices
    c = codes[:, :C].float().view(B * L, H, 128)
    s = scales[:, :H]
    deq = c * s[..., None]
    amax = deq.abs().amax(-1)
    nz = amax > 0
    assert torch.all(s[~nz] == 1.0)
    # s = amax / 448 of its dequantized values (448 s is one fp32 rounding away from the exact product)
    assert torch.allclose(s[nz], amax[nz] / 448.0, rtol=2 ** -21, atol=0)
    assert torch.all(c.abs().amax(-1)[nz] == 448.0)                 # every nonzero block holds a +-448 code
    # within one e4m3 rounding (half a step: 2^-4 relative, 2^-10 s among the subnormals) of the bf16 output, which
    # itself is one bf16 rounding of the same fp32 value
    a = bf.float().view(B * L, H, 128).abs() * (1 + 2 ** -8)
    tol = torch.maximum(2 ** -4 * a, 2 ** -10 * s[..., None]) + 2 ** -8 * a
    err = (deq - bf.float().view(B * L, H, 128)).abs()
    print(f"[fp8 attn blocks] B={B} L={L} H={H}: max |deq - bf16| / tol = {float((err / tol).max()):.3f}, "
          f"rel-L2 {rel_l2(deq.view(B * L, C), bf.float()):.3e}")
    assert torch.all(err <= tol)


def _growth_and_error(m, cfg, inp, attn):
    from oracle import mmdit_oracle as M

    m.enable_fp8(projections=True)
    if attn:
        m.enable_fp8_attention()
    got_x = []
    hooks = [b.register_forward_hook(lambda mod, a, out: got_x.append(
        torch.cat((out[1], out[0]), 1).float() if isinstance(out, tuple) else out.float()))
        for b in list(m.double_blocks) + list(m.single_blocks)]
    try:
        with torch.no_grad():
            out = m(**inp)
    finally:
        for h in hooks:
            h.remove()
    W32 = {k: v.float() for k, v in m.state_dict().items()}
    Wb = dict(m.state_dict())
    f = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    args = lambda d, dt: (d["img"], d["img_ids"], d["txt"], d["txt_ids"], d["timesteps"].to(dt), d["y_vec"])  # noqa: E731
    ref_x = []
    od, os_ = M.double_stream_block, M.single_stream_block

    def dbl(*a, **k):
        i, t = od(*a, **k)
        ref_x.append(torch.cat((t, i), 1).float())
        return i, t

    def sgl(*a, **k):
        x = os_(*a, **k)
        ref_x.append(x.float())
        return x

    M.double_stream_block, M.single_stream_block = dbl, sgl
    try:
        ref = M.model_forward(W32, cfg, *args(f, torch.float32), cond=f["cond"], guidance=f["guidance"])
    finally:
        M.double_stream_block, M.single_stream_block = od, os_
    with PR.fp8_projections(), (AR.fp8_attention() if attn else contextlib.nullcontext()):
        emu = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"], guidance=inp["guidance"].to(torch.bfloat16))
    m.disable_fp8()
    m.disable_fp8_attention()
    per_block = [rel_l2(g, r) for g, r in zip(got_x, ref_x)]
    return out, ref, emu, per_block


@pytest.mark.parametrize("attn", [False, True])
def test_full_width_mmdit_fp8_projections_against_the_oracle(attn):
    """C = 3072 (24 x 128 heads), 2 + 2 blocks, 1 x (256 text + 2304 image) tokens, every block Linear on FP8."""
    m = mmdit_model(False, True, device="cuda", **MMDIT_WIDE)
    cfg = dict(MMDIT_CFG, **MMDIT_WIDE, fused_qkv=False, use_liger_rope=True)
    inp = {k: v.cuda() for k, v in mmdit_inputs(1, 256, (1, 48, 48)).items()}
    with torch.no_grad():
        plain = m(**inp).clone()
    out, ref, emu, per_block = _growth_and_error(m, cfg, inp, attn)
    r, _ = report(f"MMDiT C=3072 2+2 blocks L=2560 FP8 projections{' + attention' if attn else ''}", out, ref)
    r_emu = rel_l2(emu, ref)
    print(f"[mmdit fp8 proj] attn={attn}: FP8-emulation reference rel_l2={r_emu:.3e}, ratio {r / r_emu:.3f}; residual "
          "stream rel_l2 after block k: " + " ".join(f"{k}:{e:.2e}" for k, e in enumerate(per_block)))
    assert torch.isfinite(out).all() and len(per_block) == cfg["depth"] + cfg["depth_single_blocks"]
    assert r <= 1.1 * r_emu, (r, r_emu)
    for k in range(1, len(per_block)):
        assert per_block[k] <= 1.3 * per_block[k - 1], (k, per_block[k - 1], per_block[k])
    with torch.no_grad():
        assert torch.equal(m(**inp), plain)   # disable_fp8 gives the bf16 bits back
