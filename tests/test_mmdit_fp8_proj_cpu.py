"""The FP8 (e4m3) projection path of MMDiT on the CPU (`enable_fp8(projections=True)`): the block-scaled output of the FP8
attention stand-in (tests/fake_osb200.py) against the block rule, the host-side model against the
FP8-emulation reference of tests/mmdit_fp8_proj_ref.py (both QKV and both RoPE layouts, with and without FP8 attention),
the launches it makes, `enable_fp8()` without the keyword, `disable_fp8()`, the adapter refusals, Ulysses sequence
parallelism on two gloo ranks and the ctypes mirror of `osb_attn_fp8_out`."""
import contextlib
import ctypes
import os

import pytest
import torch

from tests import fake_osb200 as F_
from tests import mmdit_fp8_attn_ref as AR
from tests import mmdit_fp8_proj_ref as PR
from tests.adapters import write_adapter
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn


def test_stand_in_block_output_follows_the_block_rule(fake_osb):
    """Codes and scales land in column slices of wider buffers; each (row, head) block is the block rule applied to the
    fp32 attention value, which the bf16 output of `attn_fp8` rounds."""
    B, L, H = 2, 200, 2
    qkv, kw = AR.operands_cpu(B, L, H, split=50)
    C = H * 128
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    ws = fake_osb.attn_fp8_workspace(B, L, H, "cpu")
    codes = torch.zeros(B * L, 5 * C, dtype=E4M3)
    scales = torch.full((B * L, 5 * H), -1.0)
    fake_osb.attn_fp8_blocks(q, k, v, codes[:, :C], scales[:, :H], workspace=ws, **kw)
    assert fake_osb.calls[-1][0] == "attn_fp8_blocks"
    assert not codes[:, C:].float().any() and torch.all(scales[:, H:] == -1.0)
    o = F_.attention_from_workspace(ws, B * H, L, 128 ** -0.5)
    o = o.view(B, H, L, 128).transpose(1, 2).reshape(B * L, C)
    want_codes, want_s = F_.quant_blocks(o)
    assert torch.equal(codes[:, :C].float(), want_codes.float()) and torch.equal(scales[:, :H], want_s)
    deq = (codes[:, :C].float().view(B * L, H, 128) * scales[:, :H, None]).view(B * L, C)
    amax = codes[:, :C].float().view(B * L, H, 128).abs().amax(-1)
    assert torch.all(amax == 448)                                          # every nonzero block reaches +-448
    bf = torch.zeros(B * L, C, dtype=torch.bfloat16)
    fake_osb.attn_fp8(q, k, v, bf, workspace=fake_osb.attn_fp8_workspace(B, L, H, "cpu"), **kw)
    assert rel_l2(deq, bf.float()) < 0.05                                  # within the e4m3 rounding of the bf16 output
    with pytest.raises(fake_osb.OsbError):                                     # the refusals of attn_fp8
        fake_osb.attn_fp8_blocks(q, k, v, codes[:, :C], scales[:, :H], workspace=ws, **dict(kw, Lk=100))
    with pytest.raises(fake_osb.OsbError):                                     # a scale view narrower than the heads
        fake_osb.attn_fp8_blocks(q, k, v, codes[:, :C], scales[:, :1], workspace=ws, **kw)


def _case(model, inp, attn):
    """(product, emulation reference in bf16, bf16 oracle, fp32 oracle) outputs for one model and input."""
    from oracle import mmdit_oracle as M

    cfg = dict(MMDIT_CFG, fused_qkv=model.config.fused_qkv, use_liger_rope=model.config.use_liger_rope)
    with torch.no_grad():
        out = model(**inp)
    W32 = {k: v.float() for k, v in model.state_dict().items()}
    Wb = dict(model.state_dict())
    f = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    args = lambda d, dt: (d["img"], d["img_ids"], d["txt"], d["txt_ids"], d["timesteps"].to(dt), d["y_vec"])  # noqa: E731
    ref = M.model_forward(W32, cfg, *args(f, torch.float32), cond=f["cond"], guidance=f["guidance"])
    floor = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"], guidance=inp["guidance"].to(torch.bfloat16))
    with PR.fp8_projections(), (AR.fp8_attention() if attn else contextlib.nullcontext()):
        emu = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"],
                              guidance=inp["guidance"].to(torch.bfloat16))
    return out, emu, floor, ref


@pytest.mark.parametrize("fused,liger,attn,thw", [(True, False, False, (2, 4, 6)), (False, True, False, (2, 4, 6)),
                                                  (True, True, True, (2, 4, 6)), (False, False, True, (2, 4, 6)),
                                                  (False, True, True, (1, 4, 6))],
                         ids=["True-False-False", "False-True-False", "True-True-True", "False-False-True",
                              "False-True-True-txt_len_eq_img_len"])
def test_host_mmdit_fp8_projections_follow_the_emulation(fake_osb, fused, liger, attn, thw):
    """C = 256 (2 heads of 128), 2 double + 2 single blocks, every block Linear on FP8 (and FP8 attention), against the
    fp32 oracle.  Yardstick: the emulation reference measured in the same test.  With as many text as image tokens
    (thw = (1, 4, 6)) both streams of a double block get workspaces of one shape: neither may overwrite the other's
    LN+modulate codes before its q|k|v GEMMs have read them."""
    m = mmdit_model(fused, liger)
    if attn and fused:   # the switches compose in either order
        m.enable_fp8_attention()
        m.enable_fp8(projections=True)
    else:
        m.enable_fp8(projections=True)
        if attn:
            m.enable_fp8_attention()
    inp = mmdit_inputs(thw=thw)
    with torch.no_grad():
        m(**inp)             # weights are quantized at the first forward of a CPU model
    fake_osb.reset()
    out, emu, floor, ref = _case(m, inp, attn)
    r_out, r_emu, r_bf = rel_l2(out, ref), rel_l2(emu, ref), rel_l2(floor, ref)
    print(f"[mmdit fp8 proj host] fused={fused} liger={liger} attn={attn}: product {r_out:.3e}, FP8 emulation "
          f"{r_emu:.3e}, bf16 oracle {r_bf:.3e} (rel-L2 against the fp32 oracle)")
    assert r_out < 1.1 * r_emu, (r_out, r_emu, r_bf)
    calls = list(fake_osb.calls)
    names = [c[0] for c in calls]
    nd, ns = MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"]
    assert names.count("ln_modulate") == 1                     # the final layer only: no bf16 LN pass in any block
    assert names.count("ln_modulate_fp8") == 4 * nd + ns       # mod1 + mod2 per stream, one per single block
    assert "attn_short" not in names if attn else "attn_fp8" not in names
    assert names.count("attn_fp8_blocks") == (nd + ns if attn else 0)
    quant = [c for c in calls if c[0] == "quant_blocks_fp8"]
    assert len(quant) == (0 if attn else nd + ns) and all(c[1][2] == 128 for c in quant)
    # bf16 GEMMs: embedders, the grouped modulation and the final layer; none in a block
    assert names.count("gemm") == 12 and "gemm_lora" not in names   # 9 + 1 + 2


def test_enable_fp8_without_keyword_keeps_the_mlp_path(fake_osb):
    m = mmdit_model(True, False)
    inp = mmdit_inputs(B=1)
    m.enable_fp8()
    with torch.no_grad():
        m(**inp)
        fake_osb.reset()
        mlp = m(**inp)
        mlp_calls = list(fake_osb.calls)
        m.enable_fp8(projections=True)
        m(**inp)
        fake_osb.reset()
        proj = m(**inp)
        m.enable_fp8()
        m(**inp)
        fake_osb.reset()
        again = m(**inp)
    names = [c[0] for c in mlp_calls]
    nd, ns = MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"]
    assert names.count("ln_modulate") == 2 * nd + ns + 1 and names.count("quant_blocks_fp8") == ns
    assert "attn_fp8_blocks" not in names
    assert torch.equal(again, mlp) and fake_osb.calls == mlp_calls
    assert not torch.equal(proj, mlp)


def test_disable_fp8_restores_the_bf16_bits(fake_osb):
    m, plain = mmdit_model(False, True), mmdit_model(False, True)
    inp = mmdit_inputs(B=1)
    with torch.no_grad():
        want = plain(**inp)
        plain_calls = list(fake_osb.calls)
        m.enable_fp8_attention()
        m.enable_fp8(projections=True)
        fp8 = m(**inp)
        m.disable_fp8()
        m.disable_fp8_attention()
        fake_osb.reset()
        back = m(**inp)
    assert not torch.equal(fp8, want)
    assert torch.equal(back, want) and fake_osb.calls == plain_calls
    assert m._fp8_state is None and m._fp8_proj is False


def test_fp8_proj_linears_lists_the_projections():
    m = mmdit_model(False, False)
    names = m.fp8_proj_linears()
    assert "double_blocks.0.img_attn.q_proj" in names and "double_blocks.1.txt_attn.proj" in names
    assert "single_blocks.0.k_proj" in names and "single_blocks.1.v_mlp" in names
    assert len(names) == MMDIT_CFG["depth"] * 2 * 4 + MMDIT_CFG["depth_single_blocks"] * 3
    assert mmdit_model(True, False).fp8_proj_linears()[:2] == ["double_blocks.0.img_attn.qkv",
                                                                "double_blocks.0.img_attn.proj"]


def test_adapter_refusals(fake_osb, tmp_path):
    from opensora.utils.lora import load_lora, unload_lora

    m = mmdit_model(True)
    load_lora(m, write_adapter(str(tmp_path / "a"), m, targets=["double_blocks.0.txt_attn.proj"]))
    with pytest.raises(ValueError, match="FP8 projections cannot run LoRA / DoRA adapters"):
        m.enable_fp8(projections=True)
    assert m._fp8 is False
    m.enable_fp8()            # the MLP path takes an adapter on a projection Linear
    m.disable_fp8()
    unload_lora(m)
    m.enable_fp8(projections=True)
    with pytest.raises(ValueError, match="FP8 projections, which take no LoRA"):
        load_lora(m, write_adapter(str(tmp_path / "b"), m, targets=["double_blocks.0.img_attn.proj"]))
    with pytest.raises(ValueError, match="FP8 projections, which take no LoRA"):
        load_lora(m, write_adapter(str(tmp_path / "c"), m, targets=["double_blocks.1.img_attn.qkv"]))
    load_lora(m, write_adapter(str(tmp_path / "d"), m, targets=["double_blocks.0.img_mod.lin", "final_layer.linear"]))
    inp = mmdit_inputs(B=1)
    fake_osb.reset()
    with torch.no_grad():
        out = m(**inp)
    assert "gemm_lora" in [c[0] for c in fake_osb.calls] and torch.isfinite(out.float()).all()


def _sp_worker(rank, world, port, ret):
    import sys

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests import fake_osb200

        sys.modules["osb200"] = fake_osb200
        fake_osb200.ACC_DTYPE = torch.float64   # row-local GEMMs on a row subset: no M-dependent summation-order noise
        res = []
        for fused, liger, attn in ((True, False, True), (False, True, False)):
            m = mmdit_model(fused, liger)
            m.enable_fp8(projections=True)
            if attn:
                m.enable_fp8_attention()
            inp = mmdit_inputs(B=2)
            with torch.no_grad():
                single = m(**inp)
                m.enable_sequence_parallel(dist.group.WORLD)
                sharded = m(**inp)
                m.enable_sequence_parallel(None)
            res.append(bool(torch.equal(single, sharded)))
        ret[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_mmdit_fp8_projections_ulysses_world2():
    """The inverse exchange carries e4m3 codes and per-(token, head) scales (FP8 attention) or bf16 rows quantized after
    it: split over two gloo ranks, MMDiT with FP8 projections reproduces the single-rank output bit for bit."""
    import torch.multiprocessing as mp

    port = 29500 + (os.getpid() + 73) % 2000
    ret = mp.Manager().dict()
    mp.spawn(_sp_worker, args=(2, port, ret), nprocs=2, join=True)
    for rank in (0, 1):
        assert ret.get(rank) == [True, True], ret.get(rank)


def test_attn_fp8_out_layout_matches_header():
    import subprocess
    import tempfile

    import osb200

    A = osb200.AttnFp8Out
    fields = [("sizeof(osb_attn_fp8_out)", ctypes.sizeof(A))] + [
        (f"offsetof(osb_attn_fp8_out, {n})", getattr(A, n).offset) for n in ("codes", "scales", "codes_ld", "scales_ld")]
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "probe.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "osb200.h"\nint main(){\n')
            for expr, _ in fields:
                f.write(f'printf("%zu\\n", (size_t)({expr}));\n')
            f.write("return 0;}\n")
        exe = os.path.join(d, "probe")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    for (expr, mine), theirs in zip(fields, got):
        assert mine == theirs, (expr, mine, theirs)
    assert "osb_attn_fp8_blocks" in osb200.EXPORTS
