"""LoRA / DoRA adapters on the MMDiT FP8 GEMMs on the CPU (`enable_fp8(..., lora=True)`): the stand-in of
`gemm_fp8_lora` (tests/fake_osb200.py) against its formula, the host-side model against the FP8-emulation
reference with the adapters (tests/mmdit_fp8_lora_ref.py) for LoRA and DoRA on MLP and projection targets in both QKV
and RoPE layouts, with and without FP8 projections and attention, the order of load / enable calls, unload and disable,
the e4m3 A_cat cache, the bits without an adapter, the default refusal and Ulysses sequence parallelism on two gloo ranks."""
import contextlib
import os

import pytest
import torch

from tests import fake_osb200 as F_
from tests import fp8_ref as R
from tests import mmdit_fp8_attn_ref as AR
from tests import mmdit_fp8_lora_ref as LR
from tests import mmdit_fp8_proj_ref as PR
from tests import mmdit_fp8_ref as MR
from tests.adapters import merged_state_dora, write_dora_adapter, write_adapter
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2

E4M3 = torch.float8_e4m3fn


def _mlp_targets(m):
    return m.fp8_mlp_linears()


def _block_targets(m):
    return m.fp8_mlp_linears() + m.fp8_proj_linears()


def _adapter(tmp_path, m, targets, dora, name="a", **kw):
    path = str(tmp_path / name)
    kw = dict(dict(r=12, alpha=24, rel=0.1, seed=9), **kw)
    return write_dora_adapter(path, m, targets=targets, **kw) if dora else write_adapter(path, m, targets=targets, **kw)


# ---- the stand-in ------------------------------------------------------------------------------------------------------
def test_stand_in_formula_and_col_scale(fake_osb):
    g = torch.Generator().manual_seed(0)
    M, N, K, r = 70, 256, 384, 72
    a8, sa = F_.quant_blocks(torch.randn(M, K, generator=g))
    w8, sw = F_.quant_blocks(torch.randn(N, K, generator=g), K)
    u = torch.randn(M, r, generator=g).to(torch.bfloat16)
    b = (0.1 * torch.randn(N, r, generator=g)).to(torch.bfloat16)
    bias = torch.randn(N, generator=g).to(torch.bfloat16)
    cs = 0.5 + torch.rand(N, generator=g)
    out = fake_osb.gemm_fp8_lora(a8, sa, w8, sw.view(-1), bias, u, b, col_scale=cs)
    want = cs * ((a8.float() * sa.repeat_interleave(128, 1)) @ (w8.float() * sw).t() + u.float() @ b.float().t()) + bias.float()
    assert rel_l2(out, want) < 4e-3
    ones = fake_osb.gemm_fp8_lora(a8, sa, w8, sw.view(-1), bias, u, b, col_scale=torch.ones(N))
    assert torch.equal(ones, fake_osb.gemm_fp8_lora(a8, sa, w8, sw.view(-1), bias, u, b))
    codes, scales = fake_osb.gemm_fp8_lora(a8, sa[:, 0].contiguous(), w8, sw.view(-1), bias, u, b,
                                       epilogue=F_.EPI_BIAS_GELU_TANH_FP8)
    acc = F_.gemm_fp8_lora_acc(a8, sa[:, 0].contiguous(), w8, sw.view(-1), u, b) + bias.float()
    q, s = F_.quant_blocks(torch.nn.functional.gelu(acc, approximate="tanh"))
    assert torch.equal(codes.float(), q.float()) and torch.equal(scales, s)
    with pytest.raises(fake_osb.OsbError):
        fake_osb.gemm_fp8_lora(a8, sa, w8, sw.view(-1), bias, u[:, :12], b[:, :12])   # r % 8
    assert fake_osb.calls[-1][0] == "gemm_fp8_lora"


# ---- the host model ----------------------------------------------------------------------------------------------------
def _case(model, inp, proj, attn):
    """(product, emulation reference, fp32 oracle on the merged weights g (W + s B A))."""
    from oracle import mmdit_oracle as M

    cfg = dict(MMDIT_CFG, fused_qkv=model.config.fused_qkv, use_liger_rope=model.config.use_liger_rope)
    with torch.no_grad():
        out = model(**inp)
    W32 = merged_state_dora(model)
    Wb = LR.emulation_state(model)
    f = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    args = lambda d, dt: (d["img"], d["img_ids"], d["txt"], d["txt_ids"], d["timesteps"].to(dt), d["y_vec"])  # noqa: E731
    ref = M.model_forward(W32, cfg, *args(f, torch.float32), cond=f["cond"], guidance=f["guidance"])
    with (PR.fp8_projections() if proj else MR.fp8_mlps()), (AR.fp8_attention() if attn else contextlib.nullcontext()), \
            LR.fp8_lora(model):
        emu = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"],
                              guidance=inp["guidance"].to(torch.bfloat16))
    return out, emu, ref


@pytest.mark.parametrize("fused,liger,proj,attn,dora", [(True, False, True, False, False), (False, True, True, True, True),
                                                        (True, True, False, False, True), (False, False, False, True, False),
                                                        (True, False, True, True, True)])
def test_host_mmdit_fp8_lora_follows_the_emulation(fake_osb, tmp_path, fused, liger, proj, attn, dora):
    """C = 256, 2 double + 2 single blocks, an adapter (update 30% of |W|) on every FP8 Linear, against the fp32 oracle on
    the merged weights.  Yardstick: the FP8-emulation reference with the adapters, measured in the same test."""
    m = mmdit_model(fused, liger)
    inp = mmdit_inputs()
    with torch.no_grad():
        m.enable_fp8(projections=proj)
        base = m(**inp)
        m.enable_fp8(projections=proj, lora=True)
        if attn:
            m.enable_fp8_attention()
        load_lora(m, _adapter(tmp_path, m, _block_targets(m) if proj else _mlp_targets(m), dora, rel=0.3))
        fake_osb.reset()
        out, emu, ref = _case(m, inp, proj, attn)
    r_out, r_emu = rel_l2(out, ref), rel_l2(emu, ref)
    print(f"[mmdit fp8 lora host] fused={fused} liger={liger} proj={proj} attn={attn} dora={dora}: product {r_out:.3e}, "
          f"FP8 emulation {r_emu:.3e} (rel-L2 against the fp32 oracle on merged weights)")
    assert r_out < 1.1 * r_emu, (r_out, r_emu)
    assert rel_l2(out, base.float()) > 2 * r_out, "the adapter must move the output well beyond the error"
    names = [c[0] for c in fake_osb.calls]
    nd, ns, B = MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"], inp["img"].shape[0]
    # without FP8 projections the q|k|v rows of linear1 / v_mlp (an MLP Linear) run on the bf16 LoRA GEMM
    assert names.count("gemm_lora") == (0 if proj else ns)
    if proj:   # per double block: 2 x B qkv, 2 x B proj, 2 x 2 MLP; per single block: qkv, mlp, linear2
        assert names.count("gemm_fp8_lora") == nd * (4 * B + 4) + 3 * ns
        # down GEMMs: per double block 2 qkv + 1 proj + 2 x 2 MLP; per single block linear1 (shared) + linear2
        downs = [c for c in fake_osb.calls if c[0] == "gemm_fp8_blocks" and c[1][1] % 128 != 0]
        assert len(downs) == 7 * nd + 2 * ns
    else:
        assert names.count("gemm_fp8_lora") == 4 * nd + 2 * ns


def load_lora(m, path):
    from opensora.utils.lora import load_lora as ll

    return ll(m, path)


def _forward(m, inp):
    with torch.no_grad():
        return m(**inp)


def test_call_order_unload_and_disable(fake_osb, tmp_path):
    from opensora.utils.lora import unload_lora

    inp = mmdit_inputs(B=1)
    a, b = mmdit_model(True, False), mmdit_model(True, False)
    plain = mmdit_model(True, False)
    path = _adapter(tmp_path, a, _block_targets(a), True)
    load_lora(a, path)
    a.enable_fp8(projections=True, lora=True)
    b.enable_fp8(projections=True, lora=True)
    load_lora(b, path)
    out_a, out_b = _forward(a, inp), _forward(b, inp)
    assert torch.equal(out_a, out_b)
    plain.enable_fp8(projections=True)
    want = _forward(plain, inp)
    unload_lora(a)
    fake_osb.reset()
    assert torch.equal(_forward(a, inp), want) and "gemm_fp8_lora" not in [c[0] for c in fake_osb.calls]
    b.disable_fp8()
    bf = mmdit_model(True, False)
    load_lora(bf, path)
    assert torch.equal(_forward(b, inp), _forward(bf, inp))   # back on the bf16 LoRA path


@pytest.mark.parametrize("proj", [False, True])
def test_lora_keyword_without_adapter_gives_the_fp8_bits(fake_osb, proj):
    inp = mmdit_inputs(B=1)
    a, b = mmdit_model(False, True), mmdit_model(False, True)
    a.enable_fp8(projections=proj)
    b.enable_fp8(projections=proj, lora=True)
    want = _forward(a, inp)
    calls = list(fake_osb.calls)
    fake_osb.reset()
    assert torch.equal(_forward(b, inp), want) and fake_osb.calls == calls


def test_cached_a_cat_follows_the_adapter_state(fake_osb, tmp_path):
    """An edited lora_A, lora_B or DoRA magnitude, or a reloaded adapter, reaches the FP8 path: the output equals a fresh
    model's with the same adapter state."""
    from opensora.utils.lora import unload_lora

    inp = mmdit_inputs(B=1)
    m = mmdit_model(True, False)
    m.enable_fp8(projections=True, lora=True)
    load_lora(m, _adapter(tmp_path, m, _block_targets(m), True))
    first = _forward(m, inp)
    blk = m.double_blocks[0]
    with torch.no_grad():
        blk.img_mlp[0].lora_A["default"].weight.mul_(2)
        blk.img_attn.qkv.lora_B["default"].weight.mul_(-1)
        m.single_blocks[1].linear2.lora_magnitude_vector["default"].weight.mul_(1.5)
    edited = _forward(m, inp)
    fresh = mmdit_model(True, False)
    fresh.enable_fp8(projections=True, lora=True)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    load_lora(fresh, _adapter(tmp_path, fresh, _block_targets(fresh), True, name="b"))
    fresh.load_state_dict(sd)
    assert not torch.equal(edited, first) and torch.equal(edited, _forward(fresh, inp))
    unload_lora(m)
    load_lora(m, _adapter(tmp_path, m, _block_targets(m), False, name="c", seed=4))
    other = mmdit_model(True, False)
    other.enable_fp8(projections=True, lora=True)
    load_lora(other, str(tmp_path / "c"))
    assert torch.equal(_forward(m, inp), _forward(other, inp))


def test_default_enable_fp8_still_refuses(fake_osb, tmp_path):
    m = mmdit_model(True, False)
    load_lora(m, _adapter(tmp_path, m, ["double_blocks.0.img_mlp.0"], False))
    with pytest.raises(ValueError, match="FP8 MLPs cannot run LoRA / DoRA adapters"):
        m.enable_fp8()
    n = mmdit_model(True, False)
    n.enable_fp8(projections=True)
    with pytest.raises(ValueError, match="FP8 projections, which take no LoRA"):
        load_lora(n, _adapter(tmp_path, n, ["double_blocks.0.img_attn.proj"], False, name="b"))
    n.enable_fp8(projections=True, lora=True)
    load_lora(n, str(tmp_path / "b"))
    assert torch.isfinite(_forward(n, mmdit_inputs(B=1)).float()).all()


def test_down_projection_reads_the_fp8_codes(fake_osb, tmp_path):
    """U = bf16(qdq(x) qdq_rows(A_cat)^T): the down GEMM of fc1 reads the LN+modulate codes and an A_cat quantized per
    row, whatever its rank padding."""
    m = mmdit_model(True, False)
    m.enable_fp8(lora=True)
    load_lora(m, _adapter(tmp_path, m, ["double_blocks.0.img_mlp.0"], False, r=12))
    _forward(m, mmdit_inputs(B=1))
    fp8 = m._fp8_state
    (A, q, s), = [v for k, v in fp8._la.items()]
    assert A.shape[0] == 16 and q.dtype == E4M3                              # rank 12 padded to 16
    assert torch.equal((q.float() * s[:, None]), R.dequantize(*R.quantize(A.float())).float())


def _sp_worker(rank, world, port, adapter_dir, ret):
    import sys

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests import fake_osb200

        sys.modules["osb200"] = fake_osb200
        fake_osb200.ACC_DTYPE = torch.float64   # row-local GEMMs on a row subset: no M-dependent summation-order noise
        res = []
        for fused, liger, proj, attn in ((True, False, True, True), (False, True, False, False)):
            m = mmdit_model(fused, liger)
            m.enable_fp8(projections=proj, lora=True)
            if attn:
                m.enable_fp8_attention()
            load_lora(m, adapter_dir[fused])
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
def test_mmdit_fp8_lora_ulysses_world2(tmp_path):
    """Split over two gloo ranks, MMDiT with adapters on its FP8 GEMMs reproduces the single-rank output bit for bit: the
    down projections and the adapted GEMMs are row-local."""
    import torch.multiprocessing as mp

    dirs = {}
    for fused in (True, False):
        m = mmdit_model(fused, False)
        targets = _block_targets(m) if fused else _mlp_targets(m)
        dirs[fused] = _adapter(tmp_path, m, targets, not fused, name=f"a{int(fused)}")
    port = 29500 + (os.getpid() + 91) % 2000
    ret = mp.Manager().dict()
    mp.spawn(_sp_worker, args=(2, port, dirs, ret), nprocs=2, join=True)
    for rank in (0, 1):
        assert ret.get(rank) == [True, True], ret.get(rank)
