"""The FP8 (e4m3) attention path of MMDiT on the CPU: the stand-in of tests/fake_osb200.py against the written
contract and workspace layout, the host-side MMDiTModel with `enable_fp8_attention()` against the FP8-emulation reference
of tests/mmdit_fp8_attn_ref.py (both QKV and both RoPE layouts, alone and with the FP8 MLPs), `disable_fp8_attention()`,
LoRA, the refusals, Ulysses sequence parallelism on two gloo ranks, and the ctypes mirror of `osb_attn_fp8_workspace`."""
import ctypes
import os

import pytest
import torch

from tests import fake_osb200 as F_
from tests import fp8_ref as R
from tests import mmdit_fp8_attn_ref as AR
from tests import mmdit_fp8_ref as MR
from tests.adapters import write_adapter
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn


# The S accumulator of a wgmma m64nNk32 holds, in thread (lane % 4 = t), the columns 8 j + 2 t + e of its rows; the FP8
# register A fragment wants k = 4 t + i (i < 4) and 16 + 4 t + i.  Packing the accumulator registers in order (j = 0, 1
# -> positions 4t..4t+3; j = 2, 3 -> 16 + 4t..) makes position p hold the key below.
def _accumulator_order():
    key = [0] * 32
    for t in range(4):
        cols = [2 * t, 2 * t + 1, 2 * t + 8, 2 * t + 9, 2 * t + 16, 2 * t + 17, 2 * t + 24, 2 * t + 25]
        for i, c in enumerate(cols):
            key[(i // 4) * 16 + 4 * t + i % 4] = c
    return key


def test_vt8_permutation_is_the_accumulator_order():
    want = _accumulator_order()
    assert sorted(want) == list(range(32))
    got = F_.vt8_key(torch.arange(96))
    assert got[:32].tolist() == want and got[32:64].tolist() == [32 + k for k in want]


@pytest.mark.parametrize("liger,split", [(True, 50), (False, None)])
def test_stand_in_matches_the_contract(fake_osb, liger, split):
    B, L, H = 2, 200, 2
    qkv, kw = AR.operands_cpu(B, L, H, split=split, liger=liger)
    C = H * 128
    ws = fake_osb.attn_fp8_workspace(B, L, H, "cpu")
    out = torch.zeros(B * L, C, dtype=torch.bfloat16)
    fake_osb.attn_fp8(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, workspace=ws, **kw)
    assert ws.Lpad == 256 and fake_osb.calls[-1][0] == "attn_fp8"
    skip = ("seqs_per_batch", "Lq", "Lk", "num_heads", "head_dim")
    qf, kf, vf, _ = F_.stage(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], L=L, H=H, norm_eps=1e-6,
                             **{k: v for k, v in kw.items() if k not in skip})
    # q / k: per (token, head) rows, codes = the grid rounding of x / s (tests/fp8_ref.py builds it from the e4m3 grid)
    for x, q8, s in ((qf, ws.q8, ws.s_q), (kf, ws.k8, ws.s_k)):
        rq, rs = R.quantize(x.reshape(B * H, L, 128))
        assert torch.equal(s[:, :L], rs) and torch.equal(q8[:, :L].double(), rq)
        assert torch.all(s[:, L:] == 1.0) and not q8[:, L:].float().any()          # pad rows
    # v: per channel over the sequence; vt8 holds key j(p) at position p, pad keys zero
    rv, rsv = R.quantize(vf.reshape(B * H, L, 128).transpose(1, 2))
    assert torch.equal(ws.s_v, rsv) and ws.s_v[0, 7] == 1.0
    perm = torch.tensor([32 * g + k for g in range(8) for k in _accumulator_order()])
    v8 = torch.zeros(B * H, 128, 256, dtype=torch.float64)
    v8[:, :, :L] = rv
    assert torch.equal(ws.vt8.double(), v8[:, :, perm])
    amax = ws.vt8.float().abs().amax(-1)
    assert ((amax == 448) | (amax == 0)).all() and int((amax == 0).sum()) == B   # every nonzero channel reaches +-448
    # the output: fp64 softmax attention on the dequantized workspace operands, within the P quantization
    q8, sq, k8, sk, v8k, sv = F_.workspace_operands(ws, B * H, L)
    qd, kd = q8[:, :L].double() * sq[:, :L, None], k8[:, :L].double() * sk[:, :L, None]
    vd = v8k[:, :L].double() * sv[:, None, :]
    ref = torch.softmax(qd @ kd.transpose(1, 2) / 128 ** 0.5, -1) @ vd
    emu = AR.attention_from_operands(qd.float(), kd.float(), vd.float(), 128 ** -0.5)
    got = out.view(B, L, H, 128).transpose(1, 2).reshape(B * H, L, 128)
    assert rel_l2(got, ref) < 1.1 * rel_l2(emu, ref) + 4e-3   # + the bf16 rounding of the output


def test_stand_in_refusals(fake_osb):
    qkv, kw = AR.operands_cpu(1, 64, 2)
    q, k, v = qkv[:, :256], qkv[:, 256:512], qkv[:, 512:]
    out = torch.empty(64, 256, dtype=torch.bfloat16)
    ws = fake_osb.attn_fp8_workspace(1, 64, 2, "cpu")
    for bad in (dict(head_dim=64), dict(Lk=32), dict(kv_lens=torch.tensor([3], dtype=torch.int32)),
                dict(seqs_per_batch=2)):
        with pytest.raises(fake_osb.OsbError):
            fake_osb.attn_fp8(q, k, v, out, workspace=ws, **dict(kw, **bad))
    with pytest.raises(fake_osb.OsbError):   # a workspace for fewer heads
        fake_osb.attn_fp8(q, k, v, out, workspace=fake_osb.attn_fp8_workspace(1, 64, 1, "cpu"), **kw)


def _case(model, inp, mlps=False):
    """(product, emulation reference in bf16, bf16 oracle, fp32 oracle) outputs for one model and input."""
    import contextlib

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
    with AR.fp8_attention(), (MR.fp8_mlps() if mlps else contextlib.nullcontext()):
        emu = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"],
                              guidance=inp["guidance"].to(torch.bfloat16))
    return out, emu, floor, ref


@pytest.mark.parametrize("fused,liger,mlps", [(True, False, False), (False, False, False), (False, True, False),
                                              (True, True, False), (False, True, True), (True, False, True)])
def test_host_mmdit_fp8_attention_follows_the_emulation(fake_osb, fused, liger, mlps):
    """C = 256 (2 heads of 128), 2 double + 2 single blocks, FP8 attention (and FP8 MLPs) on the stand-in, against the
    fp32 oracle.  Yardstick: the emulation reference measured in the same test."""
    m = mmdit_model(fused, liger)
    if mlps and fused:   # the two modes compose in either order
        m.enable_fp8_attention()
        m.enable_fp8()
    elif mlps:
        m.enable_fp8()
        m.enable_fp8_attention()
    else:
        m.enable_fp8_attention()
    out, emu, floor, ref = _case(m, mmdit_inputs(), mlps)
    r_out, r_emu, r_bf = rel_l2(out, ref), rel_l2(emu, ref), rel_l2(floor, ref)
    print(f"[mmdit fp8 attn host] fused={fused} liger={liger} mlps={mlps}: product {r_out:.3e}, FP8 emulation "
          f"{r_emu:.3e}, bf16 oracle {r_bf:.3e} (rel-L2 against the fp32 oracle)")
    assert r_out < 1.1 * r_emu, (r_out, r_emu, r_bf)
    names = [c[0] for c in fake_osb.calls]
    nd, ns = MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"]
    assert names.count("attn_fp8") == nd + ns and "attn_short" not in names
    assert (names.count("gemm_fp8_blocks") > 0) == mlps


def test_disable_fp8_attention_restores_the_bf16_bits(fake_osb):
    m, plain = mmdit_model(False, True), mmdit_model(False, True)
    inp = mmdit_inputs(B=1)
    with torch.no_grad():
        want = plain(**inp)
        plain_calls = list(fake_osb.calls)
        fake_osb.reset()
        m.enable_fp8_attention()
        fp8 = m(**inp)
        m.disable_fp8_attention()
        fake_osb.reset()
        back = m(**inp)
    assert not torch.equal(fp8, want)
    assert torch.equal(back, want)
    assert m._fp8_attn_state is None and fake_osb.calls == plain_calls


def test_lora_adapter_applies_with_fp8_attention(fake_osb, tmp_path):
    from opensora.utils.lora import load_lora

    m = mmdit_model(True)
    m.enable_fp8_attention()
    inp = mmdit_inputs(B=1)
    with torch.no_grad():
        base = m(**inp)
        load_lora(m, write_adapter(str(tmp_path / "a"), m, targets=["double_blocks.0.img_attn.qkv",
                                                                     "single_blocks.1.linear2"]))
        fake_osb.reset()
        adapted = m(**inp)
    names = [c[0] for c in fake_osb.calls]
    assert "gemm_lora" in names and names.count("attn_fp8") == 4
    assert not torch.equal(adapted, base) and torch.isfinite(adapted.float()).all()


def test_fp8_attention_refuses_other_head_sizes():
    from opensora.models.mmdit.model import MMDiTConfig, MMDiTModel

    cfg = dict(MMDIT_CFG, hidden_size=256, num_heads=4, axes_dim=[16, 24, 24], depth=1, depth_single_blocks=1)
    with torch.device("meta"):
        m = MMDiTModel(MMDiTConfig(from_pretrained=None, cache_dir=None, **cfg))
    with pytest.raises(ValueError, match="head size of 128"):
        m.enable_fp8_attention()
    assert m._fp8_attn is False


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
        for fused, liger in ((True, False), (False, True)):
            m = mmdit_model(fused, liger)
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
def test_mmdit_fp8_attention_ulysses_world2():
    """After the Ulysses all-to-all each rank attends over the whole sequence of its heads: split over two gloo ranks,
    MMDiT with FP8 attention reproduces the single-rank output bit for bit, in both QKV / RoPE layouts."""
    import torch.multiprocessing as mp

    port = 29500 + (os.getpid() + 41) % 2000
    ret = mp.Manager().dict()
    mp.spawn(_sp_worker, args=(2, port, ret), nprocs=2, join=True)
    for rank in (0, 1):
        assert ret.get(rank) == [True, True], ret.get(rank)


def test_attn_fp8_workspace_layout_matches_header():
    import subprocess
    import tempfile

    import osb200

    A = osb200.AttnFp8WorkspaceArgs
    fields = [("sizeof(osb_attn_fp8_workspace)", ctypes.sizeof(A))] + [
        (f"offsetof(osb_attn_fp8_workspace, {n})", getattr(A, n).offset)
        for n in ("q8", "k8", "vt8", "s_q", "s_k", "s_v", "v_amax", "capacity_bh", "capacity_lpad")]
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
