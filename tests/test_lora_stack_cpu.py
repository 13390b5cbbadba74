"""Several LoRA / DoRA adapters at once on MMDiT, on the CPU through the binding stand-in: named adapters
(`load_lora(..., adapter_name=)`), `set_adapters(model, names, weights)`, `unload_lora(model, name)`, peft-style layers
with several active adapters, FP8 with `lora=True`, Ulysses sequence parallelism and `prepare_models` with a list of
adapters.  The oracle applies peft's recursion to the weights: W_k = W_{k-1} + s_k B_k A_k for LoRA and
W_k = g_k * (W_{k-1} + s_k B_k A_k) for DoRA, g_k = m_k / ||W + s_k B_k A_k||, with s_k = scaling_k * weight_k."""
import os

import pytest
import torch
from torch import nn

from tests import mmdit_fp8_lora_ref as LR
from tests import mmdit_fp8_proj_ref as PR
from tests import mmdit_fp8_ref as MR
from tests import fp8_ref as R
from tests.adapters import load_stack, stack_registry, stacked_state, write_stack
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2


def _oracle(W32, cfg, inp):
    from oracle import mmdit_oracle as M

    f = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    return M.model_forward(W32, cfg, f["img"], f["img_ids"], f["txt"], f["txt_ids"], f["timesteps"], f["y_vec"],
                           cond=f["cond"], guidance=f["guidance"])


def _noise(W32, cfg, inp):
    from oracle import mmdit_oracle as M

    Wb = {k: v.to(torch.bfloat16) for k, v in W32.items()}
    return M.model_forward(Wb, cfg, inp["img"], inp["img_ids"], inp["txt"], inp["txt_ids"],
                           inp["timesteps"].to(torch.bfloat16), inp["y_vec"], cond=inp["cond"],
                           guidance=inp["guidance"].to(torch.bfloat16))


def _forward(m, inp):
    with torch.no_grad():
        return m(**inp)


# ---- the model with a stack on every Linear, against the oracle ---------------------------------------------------------
STACKS = {"lora_lora": (("lora", "lora"), (0.6, 1.5)),
          "lora_dora_dora": (("lora", "dora", "dora"), (1.0, 0.8, 1.25)),
          "dora_dora_lora": (("dora", "dora", "lora"), (1.25, 0.8, 1.0))}


@pytest.mark.parametrize("stack", list(STACKS))
@pytest.mark.parametrize("fused,liger", [(True, False), (False, False), (False, True)])
def test_stack_on_every_linear_vs_oracle_on_merged_weights(fake_osb, tmp_path, fused, liger, stack):
    """tests/test_lora_cpu.py's inputs and bars.  "dora_dora_lora" is "lora_dora_dora" reversed (the same three adapter
    directories, their weights reversed with them): each order matches its own oracle and is far from the other's."""
    kinds, weights = STACKS[stack]
    m = mmdit_model(fused, liger)
    inp = mmdit_inputs()
    cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
    paths = write_stack(tmp_path, mmdit_model(fused, liger), ("lora", "dora", "dora") if "dora" in stack else kinds,
                        rel=0.3 if "dora" in stack else 0.1)
    names = ["a", "b", "c"][:len(paths)]
    if stack == "dora_dora_lora":
        paths, names = paths[::-1], names[::-1]
    base = _forward(m, inp)
    load_stack(m, paths, names, weights)
    out = _forward(m, inp)
    W32 = stacked_state(m, names, weights)
    ref, noise = _oracle(W32, cfg, inp), _noise(W32, cfg, inp)
    r, rn = rel_l2(out, ref), rel_l2(noise, ref)
    assert out.shape == ref.shape
    assert r < 2e-2 and r < max(1.5 * rn, 5e-3), (r, rn)
    assert rel_l2(out, base) > 10 * r, "the stack must move the output well beyond the error"
    if "dora" in stack:
        other = _oracle(stacked_state(m, names[::-1], weights[::-1]), cfg, inp)
        assert rel_l2(out, other) > 10 * r, "the order of a stack with DoRA must matter"
    else:   # LoRA adapters commute; each weight must count
        assert rel_l2(out, _oracle(stacked_state(m, names, (1.0, 1.0)), cfg, inp)) > 10 * r


# ---- reductions to the single-adapter and plain results ----------------------------------------------------------------
def _run(fake_osb, m, inp):
    fake_osb.reset()
    out = _forward(m, inp)
    return out, list(fake_osb.calls), fake_osb.launch_count()


@pytest.mark.parametrize("fused,liger", [(True, False), (False, True)])
def test_reductions_are_bit_identical_with_the_same_launches(fake_osb, tmp_path, fused, liger):
    """A LoRA adapter "a" on every Linear and a DoRA adapter "b" on every Linear (so b also moves the modulation layers
    out of the grouped GEMM): `set_adapters([a])` gives the bits and launches of a model that holds only a,
    `set_adapters([])` those of the plain model, `unload_lora("b")` those of loading only a."""
    from opensora.utils.lora import load_lora, set_adapters, unload_lora

    inp = mmdit_inputs()
    pa, pb = write_stack(tmp_path, mmdit_model(fused, liger), ("lora", "dora"))
    only_a = load_lora(mmdit_model(fused, liger), pa)
    want_a = _run(fake_osb, only_a, inp)
    want_plain = _run(fake_osb, mmdit_model(fused, liger), inp)
    m = mmdit_model(fused, liger)
    load_lora(m, pa)
    load_lora(m, pb, adapter_name="b")
    both = _run(fake_osb, m, inp)
    assert not torch.equal(both[0], want_a[0]) and len(both[1]) > len(want_a[1])
    set_adapters(m, ["default"])
    assert _equal_runs(_run(fake_osb, m, inp), want_a)
    set_adapters(m, [])
    assert _equal_runs(_run(fake_osb, m, inp), want_plain)
    set_adapters(m, ["default", "b"])
    assert _equal_runs(_run(fake_osb, m, inp), both)
    unload_lora(m, "b")
    assert _equal_runs(_run(fake_osb, m, inp), want_a)
    assert all(set(w.lora_A) == {"default"} for w in m.modules() if hasattr(w, "base_layer"))


def _equal_runs(got, want):
    return torch.equal(got[0], want[0]) and got[1] == want[1] and got[2] == want[2] == len(want[1])


def test_unload_by_name_restores_linears_left_without_adapters(fake_osb, tmp_path):
    from opensora.utils.lora import LoraLinear, active_adapters, load_lora, unload_lora

    m = mmdit_model()
    pa, pb = write_stack(tmp_path, mmdit_model(), ("lora", "lora"), targets=["qkv", "linear1"])
    pc, = write_stack(tmp_path / "c", mmdit_model(), ("dora",), targets=["qkv", "img_in"])
    load_lora(m, pa, adapter_name="a")
    load_lora(m, pc, adapter_name="c")
    load_lora(m, pb, adapter_name="b")
    assert active_adapters(m) == ["a", "c", "b"]
    qkv = m.double_blocks[0].img_attn.qkv
    assert list(qkv.lora_A) == ["a", "c", "b"] and qkv.use_dora == {"a": False, "c": True, "b": False}
    assert "c(r=8, scaling=2.0, use_dora=True)" in repr(qkv)
    unload_lora(m, "c")
    assert type(m.img_in) is nn.Linear and isinstance(qkv, LoraLinear) and list(qkv.lora_A) == ["a", "b"]
    assert active_adapters(m) == ["a", "b"] and not len(qkv.lora_magnitude_vector)
    unload_lora(m)
    assert not any(isinstance(x, LoraLinear) for x in m.modules())


# ---- launches ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kinds", [("lora", "lora"), ("lora", "dora"), ("dora", "lora", "dora")])
def test_stack_adds_no_launch_over_one_adapter(fake_osb, tmp_path, kinds):
    """The same Linears with one adapter (of the stack's last kind, so that DoRA's modulation rule is the same) and with
    the stack: the same launch list, only the rank widths of the down GEMMs and updates differ (K = sum of the ranks)."""
    m1, m2 = mmdit_model(False, True), mmdit_model(False, True)
    inp = mmdit_inputs()
    paths = write_stack(tmp_path, mmdit_model(False, True), kinds)
    load_stack(m1, paths[-1:], ["x"])
    load_stack(m2, paths, ["a", "b", "c"][:len(paths)])
    _, one, n1 = _run(fake_osb, m1, inp)
    _, stack, n2 = _run(fake_osb, m2, inp)
    assert [c[0] for c in stack] == [c[0] for c in one] and n1 == n2 == len(one)
    ranks = sum(-(-(8 + 4 * i) // 8) * 8 for i in range(len(kinds)))
    C = MMDIT_CFG["hidden_size"]
    # the first double block's image q|k|v down GEMM: [B * Li, C] x [R, C]
    downs = [c for c in stack if c[0] == "gemm" and c[1][2] == C and c[1][1] == ranks]
    assert downs, "no down GEMM with K = sum of the ranks"


# ---- peft-style layers -------------------------------------------------------------------------------------------------
class _Mag(nn.Module):
    def __init__(self, w):
        super().__init__()
        self.weight = nn.Parameter(w)


class PeftLike(nn.Module):
    """peft's `lora.Linear` attributes only: three adapters, a LoRA "a" and DoRA "b" and "c", with their scaling folded
    in (peft's `set_scale`)."""

    def __init__(self, base, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.base_layer = base
        W = base.weight.detach().float()
        N, K = W.shape
        self.lora_A, self.lora_B = nn.ModuleDict(), nn.ModuleDict()
        self.lora_magnitude_vector = nn.ModuleDict()
        self.scaling, self.use_dora = {}, {}
        for n, r, s, dora in (("a", 8, 0.5, False), ("b", 4, 2.0, True), ("c", 12, 1.5, True)):
            A, B = torch.randn(r, K, generator=g) / K ** 0.5, torch.randn(N, r, generator=g)
            B = B * (0.3 * W.norm() / (s * B @ A).norm())   # |s B A| = 0.3 |W|
            self.lora_A[n] = nn.Linear(K, r, bias=False)
            self.lora_B[n] = nn.Linear(r, N, bias=False)
            with torch.no_grad():
                self.lora_A[n].weight.copy_(A)
                self.lora_B[n].weight.copy_(B)
            self.scaling[n], self.use_dora[n] = s, dora
            if dora:
                fac = 1 + 0.3 * (2 * torch.rand(N, generator=g) - 1)
                self.lora_magnitude_vector[n] = _Mag((W + s * B @ A).norm(dim=1) * fac)
        self.to(base.weight.dtype)
        self.active_adapters = ["a", "b", "c"]
        self.in_features, self.out_features = K, N
        self.merged = False
        self.disable_adapters = False

    weight = property(lambda self: self.base_layer.weight)
    bias = property(lambda self: self.base_layer.bias)


def peft_forward(p, x):
    """peft's `lora.Linear.forward` in eval mode, restated in fp32 (DESIGN.md 4.1c): the running result, and for a DoRA
    adapter `DoraLinearLayer.forward` with `base_result` = the running result minus the bias."""
    W, b = p.weight.float(), p.bias.float()
    result = x @ W.t() + b
    for n in p.active_adapters:
        A, B, s = p.lora_A[n].weight.float(), p.lora_B[n].weight.float(), p.scaling[n]
        lora = (x @ A.t()) @ B.t()
        if not p.use_dora[n]:
            result = result + lora * s
        else:
            g = (p.lora_magnitude_vector[n].weight.float() / torch.linalg.norm(W + s * (B @ A), dim=1)).view(1, -1)
            base_result = result - b
            result = result + (g - 1) * base_result + g * lora * s
    return result


def test_peft_style_layer_with_several_active_adapters(fake_osb):
    from opensora.models.mmdit.layers import _linear
    from opensora.utils.lora import adapter_of, adapters_of

    p = PeftLike(nn.Linear(64, 96).to(torch.bfloat16))
    x = torch.randn(37, 64, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16)
    with pytest.raises(NotImplementedError, match="3 active"):
        adapter_of(p)
    outs = {}
    for order in (["a", "b", "c"], ["c", "b", "a"], ["b", "a"]):
        p.active_adapters = order
        assert [a.name for a in adapters_of(p)] == order
        with torch.no_grad():
            out = _linear(x, p)
            want = peft_forward(p, x.float())
        r = rel_l2(out, want)
        assert r < 4e-3, (order, r)   # one bf16 rounding of the output and of c s B
        outs[tuple(order)] = (out, want)
    (o1, w1), (o2, w2) = outs[("a", "b", "c")], outs[("c", "b", "a")]
    assert rel_l2(w1, w2) > 0.05 and rel_l2(o1, w2) > 10 * rel_l2(o1, w1), "order must matter"
    p.merged = True
    assert adapters_of(p) == []


def test_weights_scale_inside_the_dora_norm(fake_osb, tmp_path):
    """One DoRA adapter with weight w equals, bit for bit, the same adapter loaded with `scale=w` (which multiplies its
    scaling): the weight reaches g = m / ||W + w s B A|| as well as the update."""
    from opensora.models.mmdit.layers import linear_parts
    from opensora.utils.lora import load_lora, set_adapters

    p, = write_stack(tmp_path, mmdit_model(), ("dora",), targets=["img_in", "linear2"])
    a, b = mmdit_model(), mmdit_model()
    load_lora(a, p, scale=0.5)
    load_lora(b, p)
    set_adapters(b, ["default"], [0.5])
    for la, lb in ((a.img_in, b.img_in), (a.single_blocks[0].linear2, b.single_blocks[0].linear2)):
        pa, pb = linear_parts(la)[2], linear_parts(lb)[2]
        assert all(torch.equal(x, y) for x, y in zip(pa, pb))
    inp = mmdit_inputs(B=1)
    assert torch.equal(_forward(a, inp), _forward(b, inp))


# ---- FP8 ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused,liger,proj", [(True, False, True), (False, True, False)])
def test_fp8_lora_stack_follows_the_emulation(fake_osb, tmp_path, fused, liger, proj):
    """tests/test_mmdit_fp8_lora_cpu.py's inputs and bar: a LoRA, DoRA, LoRA stack on every FP8 Linear, against the
    fp32 oracle on the recursively merged weights; yardstick: the FP8 emulation with the stack."""
    m = mmdit_model(fused, liger)
    inp = mmdit_inputs()
    m.enable_fp8(projections=proj, lora=True)
    base = _forward(m, inp)
    targets = m.fp8_mlp_linears() + (m.fp8_proj_linears() if proj else [])
    names, weights = ["a", "b", "c"], (1.0, 0.8, 1.25)
    load_stack(m, write_stack(tmp_path, mmdit_model(fused, liger), ("lora", "dora", "lora"), targets=targets, rel=0.3),
               names, weights)
    fake_osb.reset()
    out = _forward(m, inp)
    cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
    ref = _oracle(stacked_state(m, names, weights), cfg, inp)
    rows, ads = stack_registry(m)
    saved = MR._lin
    MR._lin = LR._lin_with(rows, ads, saved)
    try:
        from oracle import mmdit_oracle as M

        with (PR.fp8_projections() if proj else MR.fp8_mlps()):
            emu = M.model_forward(LR.emulation_state(m), cfg, inp["img"], inp["img_ids"], inp["txt"], inp["txt_ids"],
                                  inp["timesteps"].to(torch.bfloat16), inp["y_vec"], cond=inp["cond"],
                                  guidance=inp["guidance"].to(torch.bfloat16))
    finally:
        MR._lin = saved
    r_out, r_emu = rel_l2(out, ref), rel_l2(emu, ref)
    print(f"[fp8 lora stack] fused={fused} liger={liger} proj={proj}: product {r_out:.3e}, emulation {r_emu:.3e}")
    assert r_out < 1.1 * r_emu, (r_out, r_emu)
    assert rel_l2(out, base.float()) > 2 * r_out
    assert "gemm_fp8_lora" in [c[0] for c in fake_osb.calls]


def test_stacked_a_cat_quantizes_each_adapter_row_alone(fake_osb, tmp_path):
    """The e4m3 A_cat of a stack is the per-row quantization of each adapter's A, rank-padded, one after another."""
    m = mmdit_model(True, False)
    m.enable_fp8(lora=True)
    load_stack(m, write_stack(tmp_path, mmdit_model(True, False), ("lora", "dora"),
                              targets=["double_blocks.0.img_mlp.0"]), ["a", "b"])
    _forward(m, mmdit_inputs(B=1))
    (A, q, s), = [v for v in m._fp8_state._la.values()]
    lin = m.double_blocks[0].img_mlp[0]
    want = torch.zeros(8 + 16, A.shape[1])
    want[:8], want[8:20] = lin.lora_A["a"].weight.float(), lin.lora_A["b"].weight.float()
    assert torch.equal(A.float(), want)
    assert torch.equal(q.float() * s[:, None], R.dequantize(*R.quantize(want)).float())


# ---- refusals ----------------------------------------------------------------------------------------------------------
def test_refusals(fake_osb, tmp_path):
    from opensora.utils.lora import load_lora, set_adapters, unload_lora

    m = mmdit_model()
    pa, = write_stack(tmp_path / "a", mmdit_model(), ("lora",), targets=["qkv"])
    pb, = write_stack(tmp_path / "b", mmdit_model(), ("dora",), targets=["qkv", "double_blocks.0.img_mlp.0"])
    load_lora(m, pa, adapter_name="a")
    with pytest.raises(ValueError, match="already carries a LoRA adapter named 'a'"):
        load_lora(m, pb, adapter_name="a")
    load_lora(m, pb, adapter_name="b")
    with pytest.raises(ValueError, match="no adapter named 'x'"):
        set_adapters(m, ["a", "x"])
    with pytest.raises(ValueError, match="named twice"):
        set_adapters(m, ["a", "b", "a"])
    with pytest.raises(ValueError, match="2 adapters but 1 weights"):
        set_adapters(m, ["a", "b"], [0.5])
    with pytest.raises(ValueError, match="no adapter named 'x'"):
        unload_lora(m, "x")
    # FP8 MLPs without lora=True: an adapter on an MLP Linear is refused whether it is loaded or made active
    set_adapters(m, ["a"])
    m.enable_fp8(projections=False)
    with pytest.raises(ValueError, match="FP8 MLPs, which take no LoRA"):
        set_adapters(m, ["a", "b"])
    n = mmdit_model()
    n.enable_fp8(projections=True)
    with pytest.raises(ValueError, match="FP8 projections, which take no LoRA"):
        load_lora(n, pa, adapter_name="a")
    n.enable_fp8(projections=True, lora=True)
    load_stack(n, [pa, pb], ["a", "b"])
    assert torch.isfinite(_forward(n, mmdit_inputs(B=1)).float()).all()


# ---- sequence parallelism ----------------------------------------------------------------------------------------------
SP_CASES = ((True, False, (2, 24, (2, 4, 6))), (False, True, (1, 8, (1, 4, 6))))


def _sp_worker(rank, world, port, paths, ret):
    import sys

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests import fake_osb200

        sys.modules["osb200"] = fake_osb200
        fake_osb200.ACC_DTYPE = torch.float64   # row-local GEMMs on a row subset: no M-dependent summation-order noise
        res = []
        for (fused, liger, (B, Lt, thw)), ps in zip(SP_CASES, paths):
            m = mmdit_model(fused, liger)
            load_stack(m, ps, ["a", "b", "c"], (1.0, 0.8, 1.25))
            inp = mmdit_inputs(B, Lt, thw)
            with torch.no_grad():
                single = m(**inp)
                m.enable_sequence_parallel(dist.group.WORLD)
                used = m._sp_splits(Lt, thw[0] * thw[1] * thw[2]) is not None
                sharded = m(**inp)
                m.enable_sequence_parallel(None)
            res.append((bool(torch.equal(single, sharded)), used))
        ret[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_mmdit_ulysses_with_a_stack_world2(tmp_path):
    """A LoRA, DoRA, LoRA stack on every Linear: the gloo world-2 Ulysses forward reproduces the unsharded one bit for
    bit (the stand-in accumulating in fp64)."""
    import torch.multiprocessing as mp

    paths = [write_stack(tmp_path / f"c{i}", mmdit_model(fused, liger), ("lora", "dora", "lora"))
             for i, (fused, liger, _) in enumerate(SP_CASES)]
    port = 29500 + (os.getpid() + 53) % 2000
    ret = mp.Manager().dict()
    mp.spawn(_sp_worker, args=(2, port, paths, ret), nprocs=2, join=True)
    for rank in (0, 1):
        r = ret.get(rank)
        assert r is not None and all(ok and used for ok, used in r), r


# ---- prepare_models ----------------------------------------------------------------------------------------------------
def test_prepare_models_stacks_a_list_of_adapters(fake_osb, tmp_path):
    from opensora.utils import sampling as S
    from opensora.utils.lora import active_adapters
    from tests import sampling_toys as T

    pa, pb = write_stack(tmp_path, mmdit_model(), ("lora", "dora"))
    inp = mmdit_inputs(B=1)
    want = load_stack(mmdit_model(), [pa, pb], ["default", "adapter_1"], (1.0, 0.7))
    cfg = dict(model=mmdit_model(), ae=T.ToyAE(causal=True), t5=nn.Identity(), clip=nn.Identity(),
               pretrained_lora_path=[pa, (pb, 0.7)])
    m = S.prepare_models(cfg, "cpu", torch.bfloat16)[0]
    assert active_adapters(m) == ["default", "adapter_1"]
    assert m.img_in.adapter_weight == {"default": 1.0, "adapter_1": 0.7}
    assert torch.equal(_forward(m, inp), _forward(want, inp))
    one = S.prepare_models(dict(cfg, model=mmdit_model(), pretrained_lora_path=pa), "cpu", torch.bfloat16)[0]
    assert active_adapters(one) == ["default"]
