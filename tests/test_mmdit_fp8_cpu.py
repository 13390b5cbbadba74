"""The block-scaled FP8 (e4m3) MLP path of MMDiT on the CPU: the stand-in entries of tests/fake_osb200.py
against the contract arithmetic, the host-side MMDiTModel with `enable_fp8()` against the FP8-emulation reference of
tests/mmdit_fp8_ref.py (both QKV and both RoPE layouts), `disable_fp8()`, the refusals, Ulysses sequence parallelism on
two gloo ranks, and the ctypes mirror of `osb_fp8_blocks_args`."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from tests import fake_osb200 as F_
from tests import fp8_ref as R
from tests import mmdit_fp8_ref as MR
from tests.adapters import write_adapter
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn


def _blocky(seed=0, rows=6, K=512):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, K, generator=g) * torch.logspace(-3, 2, K // 128).repeat_interleave(128)
    x[1, 128:256] = 0.0          # an all-zero block: scale 1, codes 0
    x[2, 300] = -1000.0          # the block's amax lands on -448
    x[3, :128] = 3.0             # a constant block: every code is 448
    return x


def test_quant_blocks_matches_the_contract(fake_osb):
    x = _blocky().to(torch.bfloat16)
    q, s = fake_osb.quant_blocks_fp8(x)
    rq, rs = R.quantize(x.float().view(6, 4, 128))
    assert q.dtype == E4M3 and s.shape == (6, 4)
    assert torch.equal(s, rs) and torch.equal(q.double().view(6, 4, 128), rq)
    assert s[1, 1] == 1.0 and not q[1, 128:256].float().any()
    assert q[2, 300].float() == -448.0 and torch.all(q[3, :128].float() == 448.0)
    # block = K: one scale per row, any K (the weights: K = 5 x 3072 is beyond the row quantizer's 8192)
    w = torch.randn(8, 15360).to(torch.bfloat16)
    qw, sw = fake_osb.quant_blocks_fp8(w, block=15360)
    rqw, rsw = R.quantize(w.float())
    assert sw.shape == (8, 1) and torch.equal(sw[:, 0], rsw) and torch.equal(qw.double(), rqw)
    # column views of a wider buffer on both sides
    cat, cats = torch.zeros(6, 640, dtype=E4M3), torch.zeros(6, 5)
    fake_osb.quant_blocks_fp8(x[:, :256], out=cat[:, :256], out_scale=cats[:, :2])
    assert torch.equal(cat[:, :256].float(), q[:, :256].float()) and torch.equal(cats[:, :2], s[:, :2])
    with pytest.raises(fake_osb.OsbError):
        fake_osb.quant_blocks_fp8(torch.zeros(4, 200, dtype=torch.bfloat16))


@pytest.mark.parametrize("epilogue", [0, 1, 2, 5])
def test_gemm_fp8_blocks_matches_dequantized_fp32(fake_osb, epilogue):
    g = torch.Generator().manual_seed(4)
    M, N, K = 70, 256, 512
    a = _blocky(5, M, K)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    a8, sa = fake_osb.quant_blocks_fp8(a.to(torch.bfloat16))
    w8, sw = fake_osb.quant_blocks_fp8(w.to(torch.bfloat16), block=K)
    sw = sw.view(-1)
    bias = torch.randn(N, generator=g).to(torch.bfloat16)
    res = torch.randn(M, N, generator=g).to(torch.bfloat16)
    gate = torch.randn(4, N, generator=g)
    mod_index = torch.tensor([3, 1, 0, 2, 1], dtype=torch.int32)
    kw = dict(residual=res, gate=gate, group_rows=16, mod_index=mod_index) if epilogue == 2 else {}
    got = fake_osb.gemm_fp8_blocks(a8, sa, w8, sw, bias, epilogue=epilogue, **kw)
    deq_a = (a8.double().view(M, 4, 128) * sa.double()[..., None]).view(M, K)
    ref = deq_a @ (w8.double() * sw.double()[:, None]).t() + bias.double()
    if epilogue in (1, 5):
        ref = F.gelu(ref, approximate="tanh")
    elif epilogue == 2:
        gi = mod_index.long()[torch.arange(M) // 16]
        ref = ref * gate[gi].double() + res.double()
    if epilogue == 5:
        q, s = got
        assert q.dtype == E4M3 and s.shape == (M, N // 128)
        # each block's scale is amax / 448 of its values, and some code of every nonzero block is +-448
        assert torch.allclose(s, ref.abs().view(M, 2, 128).amax(-1).float() / 448, rtol=1e-5)
        assert (q.float().abs().view(M, 2, 128).amax(-1) == 448).all()
        deq = (q.double().view(M, 2, 128) * s.double()[..., None]).view(M, N)
        sb = s.double().repeat_interleave(128, dim=1)
        # within one e4m3 rounding (half a step: 2^-4 |v|, 2^-10 s among the subnormals) plus the GEMM's own error
        assert ((deq - ref).abs() <= 2.0 ** -4 * ref.abs() + 2.0 ** -10 * sb + 1e-3 * 448 * sb).all()
        return
    assert rel_l2(got, ref) < 3e-3
    if epilogue != 5:   # per-row A scales: the same value as block scales that repeat along the row
        row = fake_osb.gemm_fp8_blocks(a8, sa[:, 0].contiguous(), w8, sw, bias, epilogue=epilogue, **kw)
        rep = fake_osb.gemm_fp8_blocks(a8, sa[:, :1].expand(M, 4).contiguous(), w8, sw, bias, epilogue=epilogue, **kw)
        assert torch.equal(row, rep)
    with pytest.raises(fake_osb.OsbError):   # the FP8 GELU epilogue needs whole 128-column scale blocks
        fake_osb.gemm_fp8_blocks(a8, sa, w8[:200], sw[:200], epilogue=5)


def _fp8_case(model, inp):
    """(product with FP8, emulation reference in bf16, bf16 oracle, fp32 oracle) outputs for one model and input."""
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
    with MR.fp8_mlps():
        emu = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"],
                              guidance=inp["guidance"].to(torch.bfloat16))
    return out, emu, floor, ref


@pytest.mark.parametrize("fused,liger", [(True, False), (False, False), (False, True), (True, True)])
def test_host_mmdit_fp8_follows_the_emulation(fake_osb, fused, liger):
    """C = 256 (2 heads), 2 double + 2 single blocks, FP8 MLPs on the stand-in, against the fp32 oracle.  Yardstick: the
    FP8-emulation reference (the oracle in bf16 with its MLPs at the FP8 rounding points), measured in the same test."""
    m = mmdit_model(fused, liger)
    m.enable_fp8()
    inp = mmdit_inputs()
    out, emu, floor, ref = _fp8_case(m, inp)
    r_out, r_emu, r_bf = rel_l2(out, ref), rel_l2(emu, ref), rel_l2(floor, ref)
    print(f"[mmdit fp8 host] fused={fused} liger={liger}: product {r_out:.3e}, FP8 emulation {r_emu:.3e}, "
          f"bf16 oracle {r_bf:.3e} (rel-L2 against the fp32 oracle)")
    assert r_out < 1.1 * r_emu and r_emu > r_bf, (r_out, r_emu, r_bf)
    names = [c[0] for c in fake_osb.calls]
    nd, ns = MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"]
    assert names.count("ln_modulate_fp8") == 2 * nd + ns
    assert names.count("gemm_fp8_blocks") == 2 * (2 * nd + ns)
    # the attention output of every single block, and (first forward on the CPU) the 2 weights of every MLP
    assert names.count("quant_blocks_fp8") == ns + 2 * (2 * nd + ns)
    assert "gemm_fp8" not in names and "quant_rows_fp8" not in names
    blocks = [c[1] for c in fake_osb.calls if c[0] == "gemm_fp8_blocks"]
    assert all(d[3] == F_.EPI_BIAS_GELU_TANH_FP8 and d[4] == 1 for d in blocks[0::2])   # fc1: per-row A, FP8 out
    assert all(d[3] == 2 and d[4] == 2 for d in blocks[1::2])                          # fc2: block A, gate + residual
    assert sorted({d[2] for d in blocks[1::2]}) == [4 * 256, 5 * 256]                  # K = 4C (fc2), 5C (linear2)
    fake_osb.reset()
    with torch.no_grad():
        again = m(**inp)
    assert torch.equal(again, out)
    assert "quant_blocks_fp8" in [c[0] for c in fake_osb.calls] and \
        [c[0] for c in fake_osb.calls].count("quant_blocks_fp8") == ns   # weights stay quantized


def test_disable_fp8_restores_the_bf16_bits(fake_osb):
    m, plain = mmdit_model(False, True), mmdit_model(False, True)
    inp = mmdit_inputs(B=1)
    with torch.no_grad():
        want = plain(**inp)
        m.enable_fp8()
        fp8 = m(**inp)
        m.disable_fp8()
        fake_osb.reset()
        back = m(**inp)
    assert not torch.equal(fp8, want)
    assert torch.equal(back, want)
    assert m._fp8_state is None and not any("fp8" in c[0] for c in fake_osb.calls)


def test_fp8_refuses_sizes_beyond_the_kernels():
    """Hidden sizes or MLP widths off the 128-element block, and hidden sizes above the FP8 LN+modulate's 4096, are refused
    by enable_fp8() with the limit named.  (Meta tensors: only the shapes exist.)"""
    from opensora.models.mmdit.model import MMDiTConfig, MMDiTModel

    for hidden, heads, ratio, match in ((192, 2, 4.0, "multiples of 128"), (256, 2, 3.25, "multiples of 128"),
                                        (4224, 33, 2.0, "<= 4096")):
        cfg = dict(MMDIT_CFG, hidden_size=hidden, num_heads=heads, mlp_ratio=ratio, depth=1, depth_single_blocks=1,
                   axes_dim=[hidden // heads - 112, 56, 56])
        with torch.device("meta"):
            m = MMDiTModel(MMDiTConfig(from_pretrained=None, cache_dir=None, **cfg))
        with pytest.raises(ValueError, match=match):
            m.enable_fp8()
        assert m._fp8 is False


@pytest.mark.parametrize("fused", [True, False])
def test_fp8_and_mlp_adapters_refuse_each_other(fake_osb, tmp_path, fused):
    """LoRA / DoRA on an MLP Linear cannot run on the FP8 path: enable_fp8 on an adapted model and load_lora on an FP8
    model both refuse it.  Adapters on other Linears keep working with FP8 on."""
    from opensora.utils.lora import load_lora, unload_lora

    m = mmdit_model(fused)
    mlp_names = m.fp8_mlp_linears()
    single_mlp = "single_blocks.0." + ("linear1" if fused else "v_mlp")
    assert "double_blocks.0.img_mlp.0" in mlp_names and "single_blocks.1.linear2" in mlp_names and single_mlp in mlp_names
    for target, dora in (("double_blocks.1.txt_mlp.2", False), (single_mlp, True)):
        d = write_adapter(str(tmp_path / f"a_{target}_{dora}"), m, targets=[target], use_dora=dora)
        if dora:   # peft's DoRA export: one magnitude vector per target
            from safetensors.torch import load_file, save_file

            f = os.path.join(d, "adapter_model.safetensors")
            sd = load_file(f)
            lin = dict(m.named_modules())[target]
            sd[f"base_model.model.{target}.lora_magnitude_vector"] = lin.weight.float().norm(dim=1)
            save_file(sd, f)
        load_lora(m, d)
        with pytest.raises(ValueError, match="MLP"):
            m.enable_fp8()
        assert m._fp8 is False
        unload_lora(m)
        m.enable_fp8()
        with pytest.raises(ValueError, match="FP8"):
            load_lora(m, d)
        m.disable_fp8()
    # an adapter on the attention projections runs with FP8 MLPs
    load_lora(m, write_adapter(str(tmp_path / "proj"), m, targets=["double_blocks.0.img_attn.proj"]))
    m.enable_fp8()
    with torch.no_grad():
        out = m(**mmdit_inputs(B=1))
    assert torch.isfinite(out.float()).all()


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
            m.enable_fp8()
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
def test_mmdit_fp8_ulysses_world2():
    """The FP8 MLP path is token-local: split over two gloo ranks (Ulysses all-to-all around attention), MMDiT with FP8
    MLPs reproduces the single-rank output bit for bit, in both QKV / RoPE layouts."""
    import torch.multiprocessing as mp

    port = 29500 + (os.getpid() + 23) % 2000
    ret = mp.Manager().dict()
    mp.spawn(_sp_worker, args=(2, port, ret), nprocs=2, join=True)
    for rank in (0, 1):
        assert ret.get(rank) == [True, True], ret.get(rank)


def test_fp8_blocks_args_layout_matches_header():
    import subprocess
    import tempfile

    import osb200

    A = osb200.Fp8BlocksArgs
    fields = [("sizeof(osb_fp8_blocks_args)", ctypes.sizeof(A)),
              ("offsetof(osb_fp8_blocks_args, D8)", A.D8.offset),
              ("offsetof(osb_fp8_blocks_args, d_scale)", A.d_scale.offset),
              ("offsetof(osb_fp8_blocks_args, ldd8)", A.ldd8.offset),
              ("offsetof(osb_fp8_blocks_args, ld_dscale)", A.ld_dscale.offset),
              ("OSB_EPI_BIAS_GELU_TANH_FP8", osb200.EPI_BIAS_GELU_TANH_FP8)]
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
