"""LoRA adapters on the CPU: PEFT adapter directories written by the tests (peft itself is not a dependency) loaded by
`opensora.utils.lora.load_lora` - config semantics and every refusal -, the host-side MMDiT with an adapter on every Linear
against the fp32 oracle on the merged weights W + s B A (through the binding stand-in), Ulysses sequence parallelism, unloading, the guards of the models that take no
adapter, and the C ABI layout of osb_lora_args.  The kernel itself is checked on the GPU (tests/test_lora_gpu.py)."""
import json
import os

import pytest
import torch
from torch import nn

from tests.adapters import merged_state, write_adapter
from tests.models import MMDIT_CFG, mmdit_inputs, mmdit_model
from tests.util import rel_l2


# ---- config and format -----------------------------------------------------------------------------------------------
def test_target_modules_list_and_regex(tmp_path):
    from opensora.utils.lora import LoraLinear, load_lora, unload_lora

    m = mmdit_model()
    write_adapter(tmp_path / "list", m, targets=["qkv", "img_in", "adaLN_modulation.1"])
    load_lora(m, str(tmp_path / "list"))
    wrapped = sorted(n for n, x in m.named_modules() if isinstance(x, LoraLinear))
    want = sorted([f"double_blocks.{i}.{s}_attn.qkv" for i in range(MMDIT_CFG["depth"]) for s in ("img", "txt")]
                  + ["img_in", "final_layer.adaLN_modulation.1"])
    assert wrapped == want
    unload_lora(m)
    assert not any(isinstance(x, LoraLinear) for x in m.modules())
    write_adapter(tmp_path / "re", m, targets=r"double_blocks\.0\.(img|txt)_mod\.lin")
    load_lora(m, str(tmp_path / "re"))
    assert sorted(n for n, x in m.named_modules() if isinstance(x, LoraLinear)) == [
        "double_blocks.0.img_mod.lin", "double_blocks.0.txt_mod.lin"]
    lin = m.double_blocks[0].img_mod.lin   # peft's lora.Linear attribute layout
    assert isinstance(lin.base_layer, nn.Linear) and lin.weight is lin.base_layer.weight and lin.bias is lin.base_layer.bias
    assert set(lin.lora_A.keys()) == {"default"} and set(lin.lora_B.keys()) == {"default"} and "default" in lin.scaling


def test_rank_alpha_patterns_rslora_and_scale(tmp_path):
    from opensora.utils.lora import load_lora, unload_lora

    m = mmdit_model()
    write_adapter(tmp_path / "a", m, r=8, alpha=16, targets=["qkv", "proj", "linear2"], rank_pattern={"proj": 16},
                  alpha_pattern={r"single_blocks\.1\.linear2": 4})
    load_lora(m, str(tmp_path / "a"), scale=0.5)
    sa = m.double_blocks[0].img_attn
    assert sa.qkv.lora_A["default"].weight.shape == (8, 256) and sa.qkv.scaling["default"] == pytest.approx(0.5 * 16 / 8)
    assert sa.proj.lora_B["default"].weight.shape == (256, 16) and sa.proj.scaling["default"] == pytest.approx(0.5 * 16 / 16)
    assert m.single_blocks[0].linear2.scaling["default"] == pytest.approx(0.5 * 2.0)
    assert m.single_blocks[1].linear2.scaling["default"] == pytest.approx(0.5 * 4 / 8)
    unload_lora(m)
    write_adapter(tmp_path / "b", m, r=16, alpha=8, targets=["proj"], use_rslora=True)
    load_lora(m, str(tmp_path / "b"))
    assert m.double_blocks[1].txt_attn.proj.scaling["default"] == pytest.approx(8 / 4.0)


def test_bin_format_loads_like_safetensors(tmp_path):
    from opensora.utils.lora import adapter_of, load_lora

    m1, m2 = mmdit_model(), mmdit_model()
    write_adapter(tmp_path / "st", m1, targets=["linear1"], seed=4)
    write_adapter(tmp_path / "bin", m2, targets=["linear1"], seed=4, fmt="bin")
    load_lora(m1, str(tmp_path / "st"))
    load_lora(m2, str(tmp_path / "bin"))
    for a, b in zip(adapter_of(m1.single_blocks[0].linear1)[:2], adapter_of(m2.single_blocks[0].linear1)[:2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("change,match", [
    (dict(peft_type="IA3"), "peft_type"), (dict(use_dora=True), "use_dora"), (dict(bias="lora_only"), "bias"),
    (dict(modules_to_save=["img_in"]), "modules_to_save"), (dict(layers_to_transform=[0]), "layers_to_transform"),
    (dict(layers_pattern="blocks"), "layers_pattern"), (dict(fan_in_fan_out=True), "fan_in_fan_out"),
])
def test_config_refusals(tmp_path, change, match):
    from opensora.utils.lora import load_lora

    m = mmdit_model()
    write_adapter(tmp_path, m, targets=["qkv"], **change)
    with pytest.raises(ValueError, match=match):
        load_lora(m, str(tmp_path))


def test_target_and_tensor_refusals(tmp_path):
    from safetensors.torch import load_file, save_file

    from opensora.utils.lora import load_lora

    m = mmdit_model()
    # targets: an entry that matches nothing, a regex that matches nothing, a module that is not an nn.Linear
    for i, (tgt, match) in enumerate(((["qkv", "nope"], "'nope' matches no module"), ("nope.*", "matches no module"),
                                      (["img_norm1"], "not an nn.Linear"))):
        d = tmp_path / f"t{i}"
        write_adapter(d, m, targets=["qkv"])
        cfg = json.load(open(d / "adapter_config.json"))
        cfg["target_modules"] = tgt
        json.dump(cfg, open(d / "adapter_config.json", "w"))
        with pytest.raises(ValueError, match=match):
            load_lora(m, str(d))
    # tensors: missing, extra, mis-shaped
    d = tmp_path / "w"
    write_adapter(d, m, targets=["qkv"])
    f = str(d / "adapter_model.safetensors")
    sd = {k: v.clone() for k, v in load_file(f).items()}   # detached from the file's mapping: it is rewritten below
    key = "base_model.model.double_blocks.0.img_attn.qkv.lora_B.weight"
    for bad, match in (({k: v for k, v in sd.items() if k != key}, "miss"),
                       (dict(sd, **{"base_model.model.img_in.lora_A.weight": torch.zeros(8, 64)}), "no target uses"),
                       (dict(sd, **{key: torch.zeros(768, 4)}), "shape")):
        save_file(bad, f)
        with pytest.raises(ValueError, match=match):
            load_lora(m, str(d))
    assert not any(hasattr(x, "lora_A") for x in m.modules()), "a refused adapter must leave the model untouched"


def test_one_adapter_at_a_time_and_mmdit_only(tmp_path):
    from opensora.models.stdit.stdit3 import STDiT3_XS_2
    from opensora.utils.lora import load_lora

    m = mmdit_model()
    write_adapter(tmp_path, m, targets=["qkv"])
    load_lora(m, str(tmp_path))
    with pytest.raises(ValueError, match="already carries"):
        load_lora(m, str(tmp_path))
    with pytest.raises(TypeError, match="MMDiTModel"):
        load_lora(STDiT3_XS_2(), str(tmp_path))


# ---- the model with an adapter ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused,liger", [(True, False), (False, False), (False, True)])
def test_mmdit_adapter_on_every_linear_vs_oracle_on_merged_weights(fake_osb, tmp_path, fused, liger):
    """Same inputs and bars as tests/test_host_mmdit_cpu.py::test_mmdit_model_host_logic, every Linear adapted (update
    10% of |W|): the oracle runs on W + s B A in fp32, the noise floor is the oracle on those weights rounded to bf16."""
    from oracle import mmdit_oracle as M
    from opensora.utils.lora import load_lora

    m = mmdit_model(fused, liger)
    inp = mmdit_inputs()
    with torch.no_grad():
        base = m(**inp)
        load_lora(m, str(write_adapter(tmp_path, m, r=12, alpha=24, rel=0.1, seed=9)))
        fake_osb.reset()
        out = m(**inp)
    cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
    W32 = merged_state(m)
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
    # every token-row Linear runs on the fused kernel; the modulation stays one grouped GEMM plus one down GEMM
    names = [c[0] for c in fake_osb.calls]
    nd, ns = MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"]
    C = MMDIT_CFG["hidden_size"]
    mod_width = (2 * nd * 6 + ns * 3) * C
    assert sum(1 for c in fake_osb.calls if c[0] == "gemm" and c[1][1] == mod_width) == 1
    assert sum(1 for c in fake_osb.calls if c[0] == "gemm" and c[1][1] in (6 * C, 3 * C) and c[1][0] == 2) == 2 * nd + ns
    # per double block: 2 qkv down + 2 x B qkv, 1 proj down + 2 x B proj, 2 x (mlp0 + mlp2); per single block: 1 down,
    # qkv + mlp + linear2; embedders: img_in, cond_in, txt_in, 3 MLPEmbedders x 2, final layer x 2
    B = inp["img"].shape[0]
    want = nd * (2 * B + 2 * B + 4) + ns * 3 + 3 + 6 + 2
    assert names.count("gemm_lora") == want, (names.count("gemm_lora"), want)


def test_unload_restores_outputs_and_launches(fake_osb, tmp_path):
    from opensora.utils.lora import load_lora, unload_lora

    plain, m = mmdit_model(False, True), mmdit_model(False, True)
    inp = mmdit_inputs()
    with torch.no_grad():
        fake_osb.reset()
        want = plain(**inp)
        want_calls = list(fake_osb.calls)
        load_lora(m, str(write_adapter(tmp_path, m, seed=2)))
        adapted = m(**inp)
        unload_lora(m)
        assert all(type(x) is not type(m.img_in) or type(x) is nn.Linear for x in m.modules())
        fake_osb.reset()
        got = m(**inp)
    assert torch.equal(got, want) and not torch.equal(adapted, want)
    assert fake_osb.calls == want_calls and fake_osb.launch_count() == len(want_calls)


def test_peft_style_layer_takes_the_same_path(fake_osb):
    """A layer with peft's `lora.Linear` attributes only (active_adapters, several adapters of which one is active,
    merged / disabled flags) is read like this package's own LoraLinear."""
    from opensora.utils.lora import adapter_of

    class PeftLike(nn.Module):
        def __init__(self, base):
            super().__init__()
            self.base_layer = base
            self.lora_A = nn.ModuleDict({"a": nn.Linear(base.in_features, 8, bias=False),
                                         "b": nn.Linear(base.in_features, 4, bias=False)})
            self.lora_B = nn.ModuleDict({"a": nn.Linear(8, base.out_features, bias=False),
                                         "b": nn.Linear(4, base.out_features, bias=False)})
            self.scaling = {"a": 0.5, "b": 2.0}
            self.active_adapters = ["b"]
            self.merged = False
            self.disable_adapters = False

        weight = property(lambda self: self.base_layer.weight)
        bias = property(lambda self: self.base_layer.bias)

    p = PeftLike(nn.Linear(16, 24))
    A, B, s = adapter_of(p)
    assert A is p.lora_A["b"].weight and B is p.lora_B["b"].weight and s == 2.0
    p.merged = True
    assert adapter_of(p) is None
    p.merged, p.active_adapters = False, ["a", "b"]
    with pytest.raises(NotImplementedError, match="2 active"):
        adapter_of(p)


def test_grouped_modulation_adds_each_layer_update_into_its_slice(fake_osb, tmp_path):
    """Adapters on some modulation layers only: the grouped GEMM keeps one launch for the base weights, ONE down GEMM
    serves every adapted layer, and each layer's update is one small GEMM added into its own slice (no block-diagonal B)."""
    from opensora.utils.lora import load_lora

    m = mmdit_model()
    inp = mmdit_inputs(B=1)
    load_lora(m, str(write_adapter(tmp_path, m, targets=r".*(img_mod|modulation)\.lin", r=8, rel=0.5)))
    with torch.no_grad():
        fake_osb.reset()
        m(**inp)
    C, nd, ns = MMDIT_CFG["hidden_size"], MMDIT_CFG["depth"], MMDIT_CFG["depth_single_blocks"]
    rows1 = [c[1] for c in fake_osb.calls if c[0] == "gemm" and c[1][0] == 1]
    assert sum(1 for c in rows1 if c[1] == (2 * nd * 6 + ns * 3) * C) == 1
    assert sum(1 for c in rows1 if c[1] == (nd + ns) * 8 and c[2] == C) == 1                       # the shared down GEMM
    assert sorted(c[1] for c in rows1 if c[2] == 8 and c[3] == 2) == sorted([6 * C] * nd + [3 * C] * ns)


# ---- sequence parallelism --------------------------------------------------------------------------------------------
def _lora_sp_worker(rank, world, port, adapter_dirs, ret):
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


SP_CASES = ((True, False, (2, 24, (2, 4, 6))), (False, True, (1, 8, (1, 4, 6))))


@pytest.mark.timeout(300)
def test_mmdit_ulysses_with_adapter_world2(tmp_path):
    """With an adapter on every Linear, the gloo world-2 Ulysses forward reproduces the unsharded one bit for bit (the
    existing SP test's bar, the stand-in accumulating in fp64): LoRA is token-local."""
    import torch.multiprocessing as mp

    dirs = []
    for i, (fused, liger, _) in enumerate(SP_CASES):
        dirs.append(str(write_adapter(tmp_path / f"a{i}", mmdit_model(fused, liger), seed=i)))
    port = 29500 + (os.getpid() + 17) % 2000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_lora_sp_worker, args=(2, port, dirs, ret), nprocs=2, join=True)
    for rank in (0, 1):
        r = ret.get(rank)
        assert r is not None and all(ok and used for ok, used in r), r


# ---- models without a LoRA path -------------------------------------------------------------------------------------
def test_stdit3_and_vae_refuse_wrapped_linears(fake_osb):
    from opensora.models.stdit.stdit3 import STDiT3_XS_2
    from opensora.registry import MODELS, build_module
    from opensora.utils.lora import LoraLinear

    from opensora.utils.lora import refuse_adapters

    m = STDiT3_XS_2().to(torch.bfloat16)
    refuse_adapters(m, "STDiT3")    # clean: remembered, the next check skips the walk until some module gets wrapped
    refuse_adapters(m, "STDiT3")
    blk = m.spatial_blocks[0]
    blk.attn.proj = LoraLinear(blk.attn.proj, 8, 1.0)
    with pytest.raises(NotImplementedError, match=r"spatial_blocks\.0\.attn\.proj"):
        m(torch.zeros(1, 4, 2, 4, 4), torch.zeros(1), torch.zeros(1, 1, 300, 4096), fps=torch.ones(1),
          height=torch.ones(1), width=torch.ones(1))
    v = build_module(dict(type="hunyuan_vae", block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=4,
                          latent_channels=4), MODELS, device_map="cpu").to(torch.bfloat16)
    attn = next(x for x in v.modules() if hasattr(x, "to_q"))
    attn.to_q = LoraLinear(attn.to_q, 8, 1.0)
    with pytest.raises(NotImplementedError, match=r"to_q"):
        v.encode(torch.zeros(1, 3, 1, 16, 16))
    with pytest.raises(NotImplementedError, match=r"to_q"):
        v.decode(torch.zeros(1, 4, 1, 2, 2))


# ---- C ABI ----------------------------------------------------------------------------------------------------------
def test_lora_args_layout_matches_header():
    import ctypes
    import subprocess
    import tempfile

    import osb200

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields = [("sizeof(osb_lora_args)", ctypes.sizeof(osb200.LoraArgs))] + [
        (f"offsetof(osb_lora_args, {f})", getattr(osb200.LoraArgs, f).offset) for f in ("U", "B", "ldu", "ldb", "r", "reserved")]
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
    for (expr, mine), theirs in zip(fields, got):
        assert mine == theirs, (expr, mine, theirs)
    assert "osb_gemm_lora" in osb200.EXPORTS
