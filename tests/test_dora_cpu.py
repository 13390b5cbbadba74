"""DoRA (weight-decomposed LoRA) adapters on the CPU: PEFT DoRA adapter directories written by the tests (peft itself is
not a dependency) loaded by `opensora.utils.lora.load_lora`, the host-side MMDiT with a DoRA adapter on every Linear
against the fp32 oracle on the merged weights g * (W + s B A), peft's unmerged DoRA formula restated on one layer, the
modulation-group rule, launches, unloading, Ulysses sequence parallelism and the C ABI layout of osb_lora_args.  The
kernel itself is checked on the GPU (tests/test_dora_gpu.py)."""
import os

import pytest
import torch
from torch import nn

from tests.adapters import dora_g, merged_state_dora, write_adapter, write_dora_adapter
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2


def _mod_names(model):
    return [n for n, x in model.named_modules() if n.endswith("_mod.lin") or n.endswith("modulation.lin")]


# ---- loader ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
def test_dora_directory_loads_magnitudes(tmp_path, fmt):
    from opensora.utils.lora import DoraMagnitude, LoraLinear, adapter_of, dora_magnitude, load_lora

    m = mmdit_model()
    d = write_dora_adapter(tmp_path / fmt, m, targets=["qkv", "linear1", "img_in"], fmt=fmt)
    f = d / ("adapter_model.safetensors" if fmt == "safetensors" else "adapter_model.bin")
    if fmt == "safetensors":
        from safetensors.torch import load_file

        sd = load_file(str(f))
    else:
        sd = torch.load(str(f), weights_only=True)
    load_lora(m, str(d))
    lin = m.single_blocks[1].linear1
    assert isinstance(lin, LoraLinear) and lin.use_dora == {"default": True}
    assert isinstance(lin.lora_magnitude_vector["default"], DoraMagnitude)
    mag = dora_magnitude(lin)
    assert mag is lin.lora_magnitude_vector["default"].weight and mag.shape == (lin.out_features,)
    assert torch.equal(mag, sd["base_model.model.single_blocks.1.linear1.lora_magnitude_vector"].to(mag.dtype))
    assert adapter_of(lin)[0].shape == (8, 256)   # adapter_of keeps its (A, B, scaling) return
    assert "use_dora=True" in repr(lin)


def test_dora_missing_or_misshaped_magnitude_is_refused(tmp_path):
    from safetensors.torch import load_file, save_file

    from opensora.utils.lora import load_lora

    m = mmdit_model()
    d = write_dora_adapter(tmp_path, m, targets=["proj"])
    f = str(d / "adapter_model.safetensors")
    sd = {k: v.clone() for k, v in load_file(f).items()}
    key = "base_model.model.double_blocks.1.txt_attn.proj.lora_magnitude_vector"
    for bad, match in (({k: v for k, v in sd.items() if k != key}, "use_dora: adapter weights miss the magnitude"),
                       (dict(sd, **{key: torch.ones(255)}), r"use_dora: .* has shape \(255,\), expected \(256,\)"),
                       (dict(sd, **{key: torch.ones(256, 1)}), "use_dora: .* has shape")):
        save_file(bad, f)
        with pytest.raises(ValueError, match=match):
            load_lora(m, str(d))
    assert not any(hasattr(x, "lora_A") for x in m.modules()), "a refused adapter must leave the model untouched"
    # a magnitude vector in a plain LoRA adapter is a tensor no target uses
    import json

    cfg = json.load(open(d / "adapter_config.json"))
    cfg["use_dora"] = False
    json.dump(cfg, open(d / "adapter_config.json", "w"))
    save_file(sd, f)
    with pytest.raises(ValueError, match="no target uses"):
        load_lora(m, str(d))


def test_dora_rank_alpha_patterns_and_rslora(fake_osb, tmp_path):
    """Per-layer rank / alpha and rsLoRA set the scaling s that g = m / ||W + s B A|| reads: the packed column scale
    equals that formula on the layer's own tensors with the scaling peft would use."""
    from opensora.models.mmdit.layers import linear_parts
    from opensora.utils.lora import load_lora, unload_lora

    m = mmdit_model()
    write_dora_adapter(tmp_path / "a", m, r=8, alpha=16, targets=["qkv", "proj", "linear2"], rank_pattern={"proj": 16},
                       alpha_pattern={r"single_blocks\.1\.linear2": 4})
    load_lora(m, str(tmp_path / "a"), scale=0.5)
    sa = m.double_blocks[0].img_attn
    assert sa.proj.lora_B["default"].weight.shape == (256, 16) and sa.proj.scaling["default"] == pytest.approx(0.5)
    assert m.single_blocks[1].linear2.scaling["default"] == pytest.approx(0.5 * 4 / 8)
    for lin in (sa.qkv, sa.proj, m.single_blocks[1].linear2):
        S = linear_parts(lin)[2][2]
        assert S.dtype == torch.float32 and S.shape == (lin.out_features,)
        assert torch.allclose(S, dora_g(lin), rtol=1e-5, atol=0)
        assert (S - 1).abs().max() > 0.1
    unload_lora(m)
    write_dora_adapter(tmp_path / "b", m, r=16, alpha=8, targets=["proj"], use_rslora=True)
    load_lora(m, str(tmp_path / "b"))
    lin = m.double_blocks[1].txt_attn.proj
    assert lin.scaling["default"] == pytest.approx(8 / 4.0)
    assert torch.allclose(linear_parts(lin)[2][2], dora_g(lin), rtol=1e-5, atol=0)


# ---- one layer ---------------------------------------------------------------------------------------------------------
def test_peft_unmerged_formula_equals_merged_form(fake_osb, tmp_path):
    """peft's DoRA forward, base(x) + (g - 1) x W^T + g s (x A^T) B^T, restated in fp32 on one layer, equals the merged
    form g * x (W + s B A)^T + b that the kernel computes; the layer's forward on the stand-in is that up to bf16."""
    from opensora.utils.lora import adapter_of, dora_magnitude, load_lora

    m = mmdit_model()
    load_lora(m, str(write_dora_adapter(tmp_path, m, targets=["linear2"], rel=0.2)))
    lin = m.single_blocks[0].linear2
    A, B, s = (t.detach().float() if torch.is_tensor(t) else t for t in adapter_of(lin))
    W, b = lin.weight.detach().float(), lin.bias.detach().float()
    x = torch.randn(37, lin.in_features, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16)
    xf = x.float()
    # peft/tuners/lora/dora.py, DoraLinearLayer.forward: weight_norm over the merged weight, detached
    weight_norm = torch.linalg.norm(W + s * (B @ A), dim=1)
    g = (dora_magnitude(lin).detach().float() / weight_norm).view(1, -1)
    base_result = xf @ W.t() + b
    peft = base_result + (g - 1) * (xf @ W.t()) + g * ((xf @ A.t()) @ B.t()) * s
    merged = xf @ (g.view(-1, 1) * (W + s * (B @ A))).t() + b
    assert rel_l2(peft, merged) < 1e-5
    with torch.no_grad():
        out = lin(x)
    assert rel_l2(out, merged) < 4e-3   # one bf16 rounding
    assert rel_l2(out, xf @ (W + s * (B @ A)).t() + b) > 0.05, "g must visibly change the layer's output"


def test_peft_style_dora_layer_takes_the_same_path(fake_osb, tmp_path):
    """A layer with peft's attributes only (`use_dora`, `lora_magnitude_vector[name].weight`, several adapters of which
    one is active) gives the column scale and the output bits of this package's LoraLinear with the same tensors."""
    from opensora.models.mmdit.layers import _linear, linear_parts
    from opensora.utils.lora import dora_magnitude, load_lora

    m = mmdit_model()
    load_lora(m, str(write_dora_adapter(tmp_path, m, targets=["img_in"])))
    own = m.img_in

    class Mag(nn.Module):
        def __init__(self, w):
            super().__init__()
            self.weight = nn.Parameter(w.detach().clone())

    class PeftLike(nn.Module):
        def __init__(self, src):
            super().__init__()
            self.base_layer = src.base_layer
            A, B = src.lora_A["default"].weight, src.lora_B["default"].weight
            self.lora_A = nn.ModuleDict({"x": nn.Linear(A.shape[1], 8, bias=False), "y": nn.Linear(A.shape[1], 8, bias=False)})
            self.lora_B = nn.ModuleDict({"x": nn.Linear(8, B.shape[0], bias=False), "y": nn.Linear(8, B.shape[0], bias=False)})
            with torch.no_grad():
                self.lora_A["y"].weight.copy_(A)
                self.lora_B["y"].weight.copy_(B)
            self.lora_A.to(A.dtype), self.lora_B.to(A.dtype)
            self.scaling = {"x": 3.0, "y": src.scaling["default"]}
            self.use_dora = {"x": False, "y": True}
            self.lora_magnitude_vector = nn.ModuleDict({"y": Mag(src.lora_magnitude_vector["default"].weight)})
            self.active_adapters = ["y"]
            self.in_features, self.out_features = src.in_features, src.out_features
            self.merged = False
            self.disable_adapters = False

        weight = property(lambda self: self.base_layer.weight)
        bias = property(lambda self: self.base_layer.bias)

    p = PeftLike(own)
    assert dora_magnitude(p) is p.lora_magnitude_vector["y"].weight
    assert torch.equal(linear_parts(p)[2][2], linear_parts(own)[2][2])
    x = torch.randn(20, 64, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16)
    with torch.no_grad():
        assert torch.equal(_linear(x, p), _linear(x, own))
    p.active_adapters = ["x"]   # the active adapter is plain LoRA: no column scale
    assert dora_magnitude(p) is None and linear_parts(p)[2][2] is None


# ---- the model with a DoRA adapter -------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused,liger", [(True, False), (False, False), (False, True)])
def test_mmdit_dora_on_every_linear_vs_oracle_on_merged_weights(fake_osb, tmp_path, fused, liger):
    """tests/test_lora_cpu.py's bars, every Linear DoRA-adapted: the oracle runs on g * (W + s B A) in fp32, the noise
    floor is the oracle on those weights rounded to bf16."""
    from oracle import mmdit_oracle as M
    from opensora.utils.lora import load_lora

    m = mmdit_model(fused, liger)
    inp = mmdit_inputs()
    with torch.no_grad():
        base = m(**inp)
        load_lora(m, str(write_dora_adapter(tmp_path, m, r=12, alpha=24, rel=0.1, seed=9)))
        out = m(**inp)
    cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
    W32 = merged_state_dora(m)
    finp = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    ref = M.model_forward(W32, cfg, finp["img"], finp["img_ids"], finp["txt"], finp["txt_ids"], finp["timesteps"],
                          finp["y_vec"], cond=finp["cond"], guidance=finp["guidance"])
    Wb = {k: v.to(torch.bfloat16) for k, v in W32.items()}
    noise = M.model_forward(Wb, cfg, inp["img"], inp["img_ids"], inp["txt"], inp["txt_ids"], inp["timesteps"].to(torch.bfloat16),
                            inp["y_vec"], cond=inp["cond"], guidance=inp["guidance"].to(torch.bfloat16))
    r, rn = rel_l2(out, ref), rel_l2(noise, ref)
    assert out.shape == ref.shape
    assert r < 2e-2 and r < max(1.5 * rn, 5e-3), (r, rn)
    assert rel_l2(out, base) > 10 * r, "the adapter must move the output well beyond the error"
    # without g (the same A, B as plain LoRA) the output is far from the DoRA oracle
    W_lora = {k: v for k, v in W32.items()}
    from opensora.utils.lora import adapter_of, is_wrapped

    for name, x in m.named_modules():
        if is_wrapped(x):
            A, B, s = adapter_of(x)
            W_lora[f"{name}.weight"] = x.weight.float() + s * (B.float() @ A.float())
    ref_lora = M.model_forward(W_lora, cfg, finp["img"], finp["img_ids"], finp["txt"], finp["txt_ids"], finp["timesteps"],
                               finp["y_vec"], cond=finp["cond"], guidance=finp["guidance"])
    assert rel_l2(out, ref_lora) > 10 * r


def test_modulation_group_keeps_only_layers_without_dora(fake_osb, tmp_path):
    """DoRA on the image-stream modulation layers: they leave the grouped GEMM and each runs one down GEMM and one
    gemm_lora with its column scale; every other modulation layer stays in the group (one launch).  With DoRA on every
    modulation layer there is no grouped GEMM at all."""
    from opensora.utils.lora import load_lora, unload_lora

    m = mmdit_model()
    inp = mmdit_inputs(B=1)
    C, nd, ns = MMDIT_CFG["hidden_size"], MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"]
    load_lora(m, str(write_dora_adapter(tmp_path / "img", m, targets=r".*img_mod\.lin", r=8, rel=0.5)))
    with torch.no_grad():
        fake_osb.reset()
        m(**inp)
    rows1 = [c for c in fake_osb.calls if c[1] is not None and c[1][0] == 1]
    assert [c[1][1] for c in rows1 if c[0] == "gemm" and c[1][1] > 3 * C] == [(nd * 6 + ns * 3) * C]   # the group
    assert sorted(c[1][1] for c in rows1 if c[0] == "gemm_lora") == [6 * C] * nd
    assert sum(1 for c in rows1 if c[0] == "gemm" and c[1][1:3] == (8, C)) == nd                          # down GEMMs
    unload_lora(m)
    load_lora(m, str(write_dora_adapter(tmp_path / "all", m, targets=_mod_names(m), r=8, rel=0.5)))
    with torch.no_grad():
        fake_osb.reset()
        m(**inp)
    rows1 = [c for c in fake_osb.calls if c[1] is not None and c[1][0] == 1]
    assert not any(c[0] == "gemm" and c[1][1] > 6 * C for c in rows1)
    assert sorted(c[1][1] for c in rows1 if c[0] == "gemm_lora") == sorted([6 * C] * 2 * nd + [3 * C] * ns)


def test_dora_launches_equal_plain_lora(fake_osb, tmp_path):
    """Outside the modulation group, DoRA costs no launch: the same adapter with and without use_dora issues the same
    launch list (only the column scale differs)."""
    from opensora.utils.lora import load_lora, unload_lora

    m = mmdit_model(False, True)
    mods = set(_mod_names(m))
    targets = [n for n, x in m.named_modules() if type(x) is nn.Linear and n not in mods]
    inp = mmdit_inputs()
    with torch.no_grad():
        load_lora(m, str(write_adapter(tmp_path / "lora", m, targets=targets, seed=2)))
        fake_osb.reset()
        lora_out = m(**inp)
        lora_calls = list(fake_osb.calls)
        unload_lora(m)
        load_lora(m, str(write_dora_adapter(tmp_path / "dora", m, targets=targets, seed=2)))
        fake_osb.reset()
        dora_out = m(**inp)
    assert fake_osb.calls == lora_calls and fake_osb.launch_count() == len(lora_calls)
    assert rel_l2(dora_out, lora_out) > 0.05


def test_unload_dora_restores_outputs_and_launches(fake_osb, tmp_path):
    from opensora.utils.lora import load_lora, unload_lora

    plain, m = mmdit_model(True, False), mmdit_model(True, False)
    inp = mmdit_inputs()
    with torch.no_grad():
        fake_osb.reset()
        want = plain(**inp)
        want_calls = list(fake_osb.calls)
        load_lora(m, str(write_dora_adapter(tmp_path, m, seed=4)))
        adapted = m(**inp)
        unload_lora(m)
        assert all(type(x) is nn.Linear for x in m.modules() if hasattr(x, "weight") and isinstance(x, nn.Linear))
        fake_osb.reset()
        got = m(**inp)
    assert torch.equal(got, want) and not torch.equal(adapted, want)
    assert fake_osb.calls == want_calls and fake_osb.launch_count() == len(want_calls)


def test_pack_is_rebuilt_when_magnitude_or_base_weight_changes(fake_osb, tmp_path):
    """g reads m and W: an in-place change of either (version bump) rebuilds the cached column scale."""
    from opensora.models.mmdit.layers import linear_parts
    from opensora.utils.lora import dora_magnitude, load_lora

    m = mmdit_model()
    load_lora(m, str(write_dora_adapter(tmp_path, m, targets=["img_in"])))
    lin = m.img_in
    s0 = linear_parts(lin)[2][2]
    assert linear_parts(lin)[2][2] is s0   # cached
    with torch.no_grad():
        dora_magnitude(lin).mul_(2)
    s1 = linear_parts(lin)[2][2]
    assert torch.allclose(s1, 2 * s0, rtol=1e-6) and torch.allclose(s1, dora_g(lin), rtol=1e-5)
    with torch.no_grad():
        lin.weight.mul_(3)
    s2 = linear_parts(lin)[2][2]
    assert s2 is not s1 and torch.allclose(s2, dora_g(lin), rtol=1e-5)


# ---- sequence parallelism --------------------------------------------------------------------------------------------
SP_CASES = ((True, False, (2, 24, (2, 4, 6))), (False, True, (1, 8, (1, 4, 6))))


def _dora_sp_worker(rank, world, port, adapter_dirs, ret):
    import sys

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from opensora.utils.lora import load_lora
        from tests import fake_osb200

        sys.modules["osb200"] = fake_osb200
        fake_osb200.ACC_DTYPE = torch.float64   # row-local GEMMs on a row subset: no M-dependent summation-order noise
        res = []
        for (fused, liger, (B, Lt, thw)), d in zip(SP_CASES, adapter_dirs):
            m = mmdit_model(fused, liger)
            load_lora(m, d)
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
def test_mmdit_ulysses_with_dora_world2(tmp_path):
    """With a DoRA adapter on every Linear, the gloo world-2 Ulysses forward reproduces the unsharded one bit for bit:
    the column scale is per output channel, so it is token-local like the rest of the adapter."""
    import torch.multiprocessing as mp

    dirs = []
    for i, (fused, liger, _) in enumerate(SP_CASES):
        dirs.append(str(write_dora_adapter(tmp_path / f"a{i}", mmdit_model(fused, liger), seed=i)))
    port = 29500 + (os.getpid() + 23) % 2000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dora_sp_worker, args=(2, port, dirs, ret), nprocs=2, join=True)
    for rank in (0, 1):
        r = ret.get(rank)
        assert r is not None and all(ok and used for ok, used in r), r


# ---- C ABI ----------------------------------------------------------------------------------------------------------
def test_lora_args_layout_with_col_scale_matches_header():
    import ctypes
    import subprocess
    import tempfile

    import osb200

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = ("U", "B", "ldu", "ldb", "r", "reserved", "col_scale")
    fields = [("sizeof(osb_lora_args)", ctypes.sizeof(osb200.LoraArgs))] + [
        (f"offsetof(osb_lora_args, {f})", getattr(osb200.LoraArgs, f).offset) for f in names]
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "probe.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "osb200.h"\nint main(){\n')
            for expr, _ in fields:
                f.write(f'printf("%zu\\n", (size_t)({expr}));\n')
            f.write("return 0;}\n")
        exe = os.path.join(d, "probe")
        subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), src, "-o", exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    assert len(got) == len(fields)
    for (expr, mine), theirs in zip(fields, got):
        assert mine == theirs, (expr, mine, theirs)
    assert [n for n, _ in osb200.LoraArgs._fields_][-1] == "col_scale"
