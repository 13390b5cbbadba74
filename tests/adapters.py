"""PEFT adapter directories written by the tests (peft itself is not a dependency), the merged-weight states the
oracle runs on, and the stacked-adapter registry of the FP8 emulation."""
import json
import math
import os

import torch
from torch import nn

from tests import mmdit_fp8_lora_ref as LR


def linear_names(model):
    return [n for n, m in model.named_modules() if type(m) is nn.Linear]


def write_adapter(path, model, *, r=8, alpha=16, rel=0.1, seed=0, targets=None, fmt="safetensors", rank_pattern=None,
                  alpha_pattern=None, **cfg_extra):
    """A PEFT LoRA adapter directory for `model`: every targeted Linear gets A [r, in], B [out, r] with
    |scaling B A| = rel |W| (Frobenius), scaling as load_lora computes it for scale 1."""
    os.makedirs(path, exist_ok=True)
    targets = linear_names(model) if targets is None else targets
    cfg = dict(peft_type="LORA", r=r, lora_alpha=alpha, target_modules=targets, lora_dropout=0.05, bias="none",
               rank_pattern=rank_pattern or {}, alpha_pattern=alpha_pattern or {}, use_rslora=False, use_dora=False,
               modules_to_save=None, layers_to_transform=None, layers_pattern=None, fan_in_fan_out=False,
               task_type=None, base_model_name_or_path=None)
    cfg.update(cfg_extra)
    from opensora.utils.lora import _pattern_value, _targets

    g = torch.Generator().manual_seed(seed)
    sd = {}
    mods = dict(model.named_modules())
    for name in _targets(model, targets):
        lin = mods[name]
        rr = int(_pattern_value(cfg["rank_pattern"], name, r))
        aa = float(_pattern_value(cfg["alpha_pattern"], name, alpha))
        s = aa / math.sqrt(rr) if cfg["use_rslora"] else aa / rr
        A = torch.randn(rr, lin.in_features, generator=g) / math.sqrt(lin.in_features)
        B = torch.randn(lin.out_features, rr, generator=g)
        upd = s * B @ A
        B = B * (rel * lin.weight.detach().float().cpu().norm() / upd.norm().clamp_min(1e-30))
        sd[f"base_model.model.{name}.lora_A.weight"] = A.contiguous()
        sd[f"base_model.model.{name}.lora_B.weight"] = B.contiguous()
    with open(os.path.join(path, "adapter_config.json"), "w") as f:
        json.dump(cfg, f)
    if fmt == "safetensors":
        from safetensors.torch import save_file

        save_file(sd, os.path.join(path, "adapter_model.safetensors"))
    else:
        torch.save(sd, os.path.join(path, "adapter_model.bin"))
    return path


def merged_state(model):
    """fp32 state dict of the plain model with every adapter merged: W + scaling * B A."""
    from opensora.utils.lora import adapter_of, is_wrapped

    W = {k.replace(".base_layer.", "."): v.float() for k, v in model.state_dict().items() if ".lora_" not in k}
    with torch.no_grad():
        for name, m in model.named_modules():
            if is_wrapped(m):
                A, B, s = adapter_of(m)
                W[f"{name}.weight"] = W[f"{name}.weight"] + s * (B.float() @ A.float())
    return W


def write_dora_adapter(path, model, *, spread=0.3, mag_seed=1, fmt="safetensors", **kw):
    """A PEFT DoRA adapter directory for `model`: write_adapter's A / B plus, per target, the magnitude vector peft saves
    as `base_model.model.<name>.lora_magnitude_vector`, set to the row norms of W + s B A times a factor in
    [1 - spread, 1 + spread] so that g = m / ||W + s B A|| is well away from 1."""
    write_adapter(path, model, fmt=fmt, use_dora=True, **kw)
    cfg = json.load(open(os.path.join(path, "adapter_config.json")))
    f = os.path.join(path, "adapter_model.safetensors" if fmt == "safetensors" else "adapter_model.bin")
    if fmt == "safetensors":
        from safetensors.torch import load_file, save_file

        sd = {k: v.clone() for k, v in load_file(f).items()}
    else:
        sd = torch.load(f, weights_only=True)
    from opensora.utils.lora import _pattern_value

    g = torch.Generator().manual_seed(mag_seed)
    mods = dict(model.named_modules())
    for k in [k for k in sd if k.endswith(".lora_A.weight")]:
        name = k[len("base_model.model."):-len(".lora_A.weight")]
        lin = mods[name]
        r = int(_pattern_value(cfg["rank_pattern"], name, cfg["r"]))
        a = float(_pattern_value(cfg["alpha_pattern"], name, cfg["lora_alpha"]))
        s = a / math.sqrt(r) if cfg["use_rslora"] else a / r
        W = lin.weight.detach().float().cpu() + s * sd[f"base_model.model.{name}.lora_B.weight"] @ sd[k]
        fac = 1 + spread * (2 * torch.rand(lin.out_features, generator=g) - 1)
        sd[f"base_model.model.{name}.lora_magnitude_vector"] = (W.norm(dim=1) * fac).contiguous()
    if fmt == "safetensors":
        save_file(sd, f)
    else:
        torch.save(sd, f)
    return path


def dora_g(lin):
    """g = m / ||W + s B A||_2 per output row, fp32, from the layer's own (bf16) tensors."""
    from opensora.utils.lora import adapter_of, dora_magnitude

    A, B, s = adapter_of(lin)
    with torch.no_grad():
        W = lin.weight.float() + s * (B.float() @ A.float())
        return dora_magnitude(lin).float() / W.norm(dim=1)


def merged_state_dora(model):
    """fp32 state dict of the plain model with every adapter merged: g * (W + s B A) for DoRA layers (bias untouched),
    W + s B A for plain LoRA layers."""
    from opensora.utils.lora import adapter_of, dora_magnitude, is_wrapped

    W = {k.replace(".base_layer.", "."): v.float() for k, v in model.state_dict().items()
         if ".lora_" not in k}
    with torch.no_grad():
        for name, m in model.named_modules():
            if is_wrapped(m):
                A, B, s = adapter_of(m)
                w = W[f"{name}.weight"] + s * (B.float() @ A.float())
                if dora_magnitude(m) is not None:
                    w = dora_g(m)[:, None] * w
                W[f"{name}.weight"] = w
    return W


def write_stack(tmp_path, model, kinds, targets=None, **kw):
    """One adapter directory per entry of `kinds` ("lora" / "dora"), all written from the plain `model` with their own
    seeds; returns the paths."""
    targets = linear_names(model) if targets is None else targets
    paths = []
    for i, kind in enumerate(kinds):
        path = tmp_path / f"{kind}{i}"
        args = dict(dict(r=8 + 4 * i, alpha=16, rel=0.1, seed=20 + i, targets=targets), **kw)
        if kind == "dora":
            write_dora_adapter(path, model, mag_seed=30 + i, **args)
        else:
            write_adapter(path, model, **args)
        paths.append(str(path))
    return paths


def load_stack(model, paths, names, weights=None):
    from opensora.utils.lora import load_lora, set_adapters

    for p, n in zip(paths, names):
        load_lora(model, p, adapter_name=n)
    return set_adapters(model, names, weights)


def stacked_state(model, names, weights):
    """fp32 state dict of the plain model with the adapters `names` (in that order, with `weights`) merged by peft's
    recursion, read from each layer's own lora_A / lora_B / scaling / magnitude tensors."""
    from opensora.utils.lora import is_wrapped

    W = {k.replace(".base_layer.", "."): v.float() for k, v in model.state_dict().items() if ".lora_" not in k}
    with torch.no_grad():
        for name, m in model.named_modules():
            if not is_wrapped(m):
                continue
            W0 = m.weight.float()
            w = W0
            for n, wt in zip(names, weights):
                if n not in m.lora_A:
                    continue
                upd = m.scaling[n] * wt * (m.lora_B[n].weight.float() @ m.lora_A[n].weight.float())
                w = w + upd
                if m.use_dora[n]:
                    w = (m.lora_magnitude_vector[n].weight.float() / (W0 + upd).norm(dim=1))[:, None] * w
            W[f"{name}.weight"] = w
    return W


def stack_registry(model):
    """tests/mmdit_fp8_lora_ref.py's registry for stacks: per adapted Linear the unrolled form of the recursion,
    A_cat = the A_k one after another, bf16(c_k s_k B_k) side by side and G, c_k = 1 / the product of the g_j of the DoRA
    adapters before k, G = the product of all of them."""
    from opensora.utils.lora import adapters_of, is_wrapped

    rows, ads = {}, []
    with torch.no_grad():
        for _, m in model.named_modules():
            stack = adapters_of(m) if is_wrapped(m) else []
            if not stack:
                continue
            W = m.weight.float()
            G = torch.ones(W.shape[0], device=W.device)
            As, Bs = [], []
            for ad in stack:
                upd = ad.scaling * (ad.B.float() @ ad.A.float())
                As.append(ad.A.float())
                Bs.append(((ad.scaling / G)[:, None] * ad.B.float()).to(torch.bfloat16).float())
                if ad.magnitude is not None:
                    G = G * ad.magnitude.float() / (W + upd).norm(dim=1)
            ads.append((torch.cat(As), torch.cat(Bs, 1), G))
            for i, k in enumerate(LR._row_keys(m.weight)):
                rows[k] = (len(ads) - 1, i)
    return rows, ads
