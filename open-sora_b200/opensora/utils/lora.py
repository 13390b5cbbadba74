"""LoRA adapters for MMDiT inference, kept unmerged as the reference keeps them (`PeftModel.from_pretrained(model, path,
is_trainable=False)`, opensora/utils/sampling.py:542-545).

`load_lora(model, path)` reads a PEFT adapter directory (adapter_config.json + adapter_model.safetensors / .bin) and
replaces every targeted `nn.Linear` with a `LoraLinear`, which has the attribute layout of peft's `lora.Linear`
(`base_layer`, `lora_A` / `lora_B` ModuleDicts with a "default" entry, `scaling["default"]`, `weight` / `bias` of the
base layer).  The MMDiT processors read any Linear through `adapter_of`, so a model wrapped by peft itself takes the
same path.  The forward computes x W^T + (x A^T)(s B)^T in one fp32 accumulator (osb_gemm_lora): merging s B A into the
bf16 weight instead would round most of a small update away, and switching or removing an adapter would rewrite the
base weights.

Restated from peft's LoraConfig semantics (peft is not a dependency): `target_modules` as a list matches a module whose
name equals an entry or ends with "." + entry, as a string it is a regex full match; `rank_pattern` / `alpha_pattern`
keys match a module name that ends with the pattern (regex) at a "." boundary; scaling = lora_alpha / r, or
lora_alpha / sqrt(r) with `use_rslora`, times `scale`.  `lora_dropout` is inference-irrelevant and ignored.

DoRA (`use_dora`, weight-decomposed LoRA): peft's forward is base(x) + (g - 1) x W^T + g s x A^T B^T with
g = m / ||W + s B A||_2 per output row (m = `lora_magnitude_vector`), i.e. g * (x W^T + s x A^T B^T) + bias.  g is
computed once per pack, in fp32 on the weights' device, and the kernel multiplies its accumulator by it before the bias
(osb_lora_args.col_scale).  Everything else an adapter could ask for (trained biases, modules_to_save, layer selection,
fan_in_fan_out) is refused."""
from __future__ import annotations

import json
import math
import os
import re
import weakref

import torch
from torch import nn

ADAPTER = "default"


class DoraMagnitude(nn.Module):
    """peft's `DoraLinearLayer` as far as inference reads it: the magnitude vector m [out_features] as `.weight`."""

    def __init__(self, out_features: int, device=None, dtype=None):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(out_features, device=device, dtype=dtype))


class LoraLinear(nn.Module):
    """An `nn.Linear` with one unmerged low-rank adapter, in peft's `lora.Linear` attribute layout (with DoRA:
    `use_dora[name]` and `lora_magnitude_vector[name].weight`)."""

    def __init__(self, base: nn.Linear, r: int, scaling: float, use_dora: bool = False):
        super().__init__()
        self.base_layer = base
        kw = dict(bias=False, device=base.weight.device, dtype=base.weight.dtype)
        self.lora_A = nn.ModuleDict({ADAPTER: nn.Linear(base.in_features, r, **kw)})
        self.lora_B = nn.ModuleDict({ADAPTER: nn.Linear(r, base.out_features, **kw)})
        self.scaling = {ADAPTER: float(scaling)}
        self.use_dora = {ADAPTER: bool(use_dora)}
        self.lora_magnitude_vector = nn.ModuleDict(
            {ADAPTER: DoraMagnitude(base.out_features, base.weight.device, base.weight.dtype)} if use_dora else {})
        self.active_adapters = [ADAPTER]
        self.in_features, self.out_features = base.in_features, base.out_features

    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return self.base_layer.bias

    def forward(self, x):
        from opensora.models.mmdit.layers import _linear

        return _linear(x.reshape(-1, x.shape[-1]).contiguous(), self).view(*x.shape[:-1], self.out_features)

    def extra_repr(self) -> str:
        dora = ", use_dora=True" if self.use_dora[ADAPTER] else ""
        return f"r={self.lora_A[ADAPTER].out_features}, scaling={self.scaling[ADAPTER]}{dora}"


def is_wrapped(module: nn.Module) -> bool:
    """True for a LoRA-wrapped Linear, this module's or peft's."""
    return hasattr(module, "base_layer") and hasattr(module, "lora_A")


def _active(lin: nn.Module):
    """Name of the active adapter of a LoRA-wrapped Linear, or None (plain Linear, adapters disabled or merged)."""
    la = getattr(lin, "lora_A", None)
    if la is None or getattr(lin, "merged", False) or getattr(lin, "disable_adapters", False):
        return None
    names = [n for n in getattr(lin, "active_adapters", list(la.keys())) if n in la]
    if not names:
        return None
    if len(names) > 1:
        raise NotImplementedError(f"{len(names)} active LoRA adapters on one Linear: osb200 runs one at a time")
    return names[0]


def adapter_of(lin: nn.Module):
    """(A [r, in], B [out, r], scaling) of the active adapter of a LoRA-wrapped Linear, or None for a plain Linear (and
    for a peft layer whose adapters are disabled or already merged into the base weight).  A DoRA adapter also has a
    magnitude vector: `dora_magnitude`."""
    n = _active(lin)
    if n is None:
        return None
    return lin.lora_A[n].weight, lin.lora_B[n].weight, float(lin.scaling[n])


def dora_magnitude(lin: nn.Module):
    """The magnitude vector m [out_features] of the active adapter when it is a DoRA adapter, else None."""
    n = _active(lin)
    if n is None or not getattr(lin, "use_dora", {}).get(n, False):
        return None
    return lin.lora_magnitude_vector[n].weight


def _state(lins):
    """What a packed adapter depends on: identity and version of every A / B tensor and the scaling; for DoRA also of
    the magnitude vector and the base weight, which g = m / ||W + s B A|| reads."""
    out = []
    for lin in lins:
        ad = adapter_of(lin)
        if ad is None:
            out.append(None)
            continue
        st = (id(lin), ad[0].data_ptr(), ad[0]._version, ad[1].data_ptr(), ad[1]._version, ad[2], ad[0].dtype, ad[0].device)
        m = dora_magnitude(lin)
        if m is not None:
            st += (m.data_ptr(), m._version, lin.weight.data_ptr(), lin.weight._version)
        out.append(st)
    return tuple(out)


_PACKS = weakref.WeakKeyDictionary()   # first Linear of a pack -> {layout: (adapter state, pack)}


def lora_pack(groups, k_pad: int = 0):
    """The adapters of Linears that read ONE input, for one down GEMM: `groups` lists, per weight the forward multiplies
    that input with, its output rows as (linear, row_lo, row_hi) slices (a packed q|k|v weight has three; linear1's qkv
    part is (linear1, 0, 3C)).  Returns None when no member carries an adapter, else
    (A_cat, [B_cat or None per group], [col_scale or None per group]): A_cat bf16 [R, K + k_pad] stacks every adapted
    member's A once (rank zero-padded to a multiple of 8, K zero-padded by k_pad like the base weight); B_cat bf16
    [rows, R] holds scaling * B in the member's rows and rank columns and zeros elsewhere, None for a group without an
    adapted member; col_scale fp32 [rows] holds DoRA's g = m / ||W + s B A|| in a DoRA member's rows and 1.0 elsewhere,
    None for a group without a DoRA member.  Cached on the adapter state."""
    lins = []
    for g in groups:
        for lin, _, _ in g:
            if all(lin is not l for l in lins):
                lins.append(lin)
    state = _state(lins)
    if all(s is None for s in state):
        return None
    key = (tuple(tuple((id(l), lo, hi) for l, lo, hi in g) for g in groups), k_pad)
    ent = _PACKS.setdefault(lins[0], {})
    hit = ent.get(key)
    if hit is None or hit[0] != state:
        ent[key] = hit = (state, _build_pack(groups, lins, k_pad))
    return hit[1]


def _build_pack(groups, lins, k_pad):
    ads = {id(l): adapter_of(l) for l in lins}
    offs, R = {}, 0
    for lin in lins:
        if ads[id(lin)] is not None:
            offs[id(lin)] = R
            R += -(-ads[id(lin)][0].shape[0] // 8) * 8
    ref = next(a for a in ads.values() if a is not None)[0]
    K = ref.shape[1]
    with torch.no_grad():
        A_cat = torch.zeros(R, K + k_pad, dtype=torch.bfloat16, device=ref.device)
        for lin in lins:
            if ads[id(lin)] is not None:
                A = ads[id(lin)][0]
                A_cat[offs[id(lin)]:offs[id(lin)] + A.shape[0], :K] = A
        Bs = []
        for g in groups:
            if all(ads[id(l)] is None for l, _, _ in g):
                Bs.append(None)
                continue
            Bg = torch.zeros(sum(hi - lo for _, lo, hi in g), R, dtype=torch.float32, device=ref.device)
            row = 0
            for lin, lo, hi in g:
                if ads[id(lin)] is not None:
                    A, Bw, s = ads[id(lin)]
                    o = offs[id(lin)]
                    Bg[row:row + hi - lo, o:o + A.shape[0]] = s * Bw[lo:hi].float()
                row += hi - lo
            Bs.append(Bg.to(torch.bfloat16).contiguous())   # bf16(s B): the scale is folded once per load / change
        gs = {id(l): _dora_scale(l, *ads[id(l)]) for l in lins if ads[id(l)] is not None and dora_magnitude(l) is not None}
        Ss = []
        for g in groups:
            if all(id(l) not in gs for l, _, _ in g):
                Ss.append(None)
                continue
            Ss.append(torch.cat([gs[id(l)][lo:hi] if id(l) in gs else torch.ones(hi - lo, device=ref.device)
                                 for l, lo, hi in g]).contiguous())
    return A_cat, Bs, Ss


_NORM_CHUNK = 1 << 24   # fp32 elements of W + s B A materialised at a time while g is computed (64 MB)


def _dora_scale(lin, A, B, s):
    """g = m / ||W + s B A||_2 over in_features, fp32 [out_features], on the weights' device; computed in row chunks so
    the temporary stays bounded whatever the layer's size.  (peft's DoRA layer recomputes this on every forward.)"""
    W = lin.weight
    Af = A.float()
    norm = torch.empty(W.shape[0], dtype=torch.float32, device=W.device)
    step = max(1, _NORM_CHUNK // W.shape[1])
    for lo in range(0, W.shape[0], step):
        hi = min(lo + step, W.shape[0])
        norm[lo:hi] = torch.linalg.vector_norm(W[lo:hi].float() + s * (B[lo:hi].float() @ Af), dim=1)
    return dora_magnitude(lin).float() / norm


# LoRA-wrapped modules registered into any parent module since import.  Wrapping (peft's and load_lora's) assigns the
# wrapper to its parent, which runs torch's global registration hooks: while the count stands still, no model can have
# gained an adapter, and refuse_adapters need not walk the module tree again (about 1 ms for STDiT3-XL, every step).
_WRAPS = [0]


def _count_wraps(module, name, submodule):
    if submodule is not None and is_wrapped(submodule):
        _WRAPS[0] += 1


torch.nn.modules.module.register_module_module_registration_hook(_count_wraps)


def refuse_adapters(model: nn.Module, what: str) -> None:
    """Models whose forward does not apply adapters raise instead of silently computing the base model."""
    if model.__dict__.get("_osb_lora_checked") == _WRAPS[0]:
        return
    for name, m in model.named_modules():
        if is_wrapped(m):
            raise NotImplementedError(f"{what}: module '{name}' carries a LoRA adapter, but LoRA is implemented for the "
                                      "MMDiT denoiser only; unload it or merge it into the weights")
    model.__dict__["_osb_lora_checked"] = _WRAPS[0]


# ---- PEFT adapter directories ---------------------------------------------------------------------------------------
def _read_config(path: str) -> dict:
    with open(os.path.join(path, "adapter_config.json")) as f:
        cfg = json.load(f)
    if cfg.get("peft_type", "LORA") != "LORA":
        raise ValueError(f"peft_type {cfg.get('peft_type')!r} is not supported: only LORA adapters can be loaded")
    if cfg.get("bias", "none") != "none":
        raise ValueError(f"bias={cfg['bias']!r}: adapters with trained biases are not supported (only bias='none')")
    if cfg.get("modules_to_save"):
        raise ValueError(f"modules_to_save={cfg['modules_to_save']!r}: fully trained module copies are not supported")
    for k in ("layers_to_transform", "layers_pattern"):
        if cfg.get(k) not in (None, [], ""):
            raise ValueError(f"{k}={cfg[k]!r}: layer selection is not supported")
    if cfg.get("fan_in_fan_out"):
        raise ValueError("fan_in_fan_out: transposed (Conv1D) weights are not supported")
    if not cfg.get("target_modules"):
        raise ValueError("adapter_config.json names no target_modules")
    return cfg


def _read_weights(path: str) -> dict:
    st = os.path.join(path, "adapter_model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file

        return load_file(st)
    bn = os.path.join(path, "adapter_model.bin")
    if os.path.exists(bn):
        return torch.load(bn, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"{path} holds neither adapter_model.safetensors nor adapter_model.bin")


def _targets(model: nn.Module, target_modules) -> list[str]:
    names = [n for n, _ in model.named_modules() if n]
    if isinstance(target_modules, str):
        hit = [n for n in names if re.fullmatch(target_modules, n)]
        if not hit:
            raise ValueError(f"target_modules regex {target_modules!r} matches no module of the model")
        return hit
    hit = []
    for t in target_modules:
        sel = [n for n in names if n == t or n.endswith("." + t)]
        if not sel:
            raise ValueError(f"target_modules entry {t!r} matches no module of the model")
        hit += [n for n in sel if n not in hit]
    return [n for n in names if n in hit]


def _pattern_value(patterns: dict, name: str, default):
    for p, v in (patterns or {}).items():
        if re.match(rf"(.*\.)?({p})$", name):
            return v
    return default


def load_lora(model: nn.Module, path: str, scale: float = 1.0) -> nn.Module:
    """Load the PEFT LoRA adapter in directory `path` into the MMDiT `model`, in place, unmerged; `scale` multiplies
    every layer's scaling (lora_alpha / r).  A DoRA adapter (`use_dora: true`) also carries one magnitude vector per
    target, saved by peft as `base_model.model.<name>.lora_magnitude_vector` [out_features] (its state-dict export drops
    the adapter name and the DoRA layer's `.weight`).  Returns the model.  One adapter at a time: `unload_lora` first."""
    from opensora.models.mmdit.model import MMDiTModel

    if not isinstance(model, MMDiTModel):
        raise TypeError(f"load_lora supports MMDiTModel only, got {type(model).__name__}")
    for name, m in model.named_modules():
        if is_wrapped(m):
            raise ValueError(f"the model already carries a LoRA adapter (at '{name}'): unload_lora first")
    cfg = _read_config(path)
    weights = _read_weights(path)
    prefix = "base_model.model."
    r0, alpha0 = int(cfg.get("r", 8)), float(cfg.get("lora_alpha", 8))
    dora = bool(cfg.get("use_dora"))
    mods = dict(model.named_modules())
    plan, used = [], set()
    for name in _targets(model, cfg["target_modules"]):
        lin = mods[name]
        if type(lin) is not nn.Linear:
            raise ValueError(f"target module '{name}' is a {type(lin).__name__}, not an nn.Linear")
        r = int(_pattern_value(cfg.get("rank_pattern"), name, r0))
        alpha = float(_pattern_value(cfg.get("alpha_pattern"), name, alpha0))
        s = (alpha / math.sqrt(r) if cfg.get("use_rslora") else alpha / r) * scale
        ka, kb = f"{prefix}{name}.lora_A.weight", f"{prefix}{name}.lora_B.weight"
        for k, shape in ((ka, (r, lin.in_features)), (kb, (lin.out_features, r))):
            if k not in weights:
                raise ValueError(f"adapter weights miss {k}")
            if tuple(weights[k].shape) != shape:
                raise ValueError(f"{k} has shape {tuple(weights[k].shape)}, expected {shape} (r = {r})")
        used |= {ka, kb}
        mag = None
        if dora:
            km = f"{prefix}{name}.lora_magnitude_vector"
            if km not in weights:
                raise ValueError(f"use_dora: adapter weights miss the magnitude vector {km}")
            if tuple(weights[km].shape) != (lin.out_features,):
                raise ValueError(f"use_dora: {km} has shape {tuple(weights[km].shape)}, expected ({lin.out_features},)")
            used.add(km)
            mag = weights[km]
        plan.append((name, lin, r, s, weights[ka], weights[kb], mag))
    if getattr(model, "_fp8", False) and not getattr(model, "_fp8_lora", False):
        on_mlp = sorted({p[0] for p in plan} & set(model.fp8_mlp_linears()))
        if on_mlp:
            raise ValueError(f"the model runs FP8 MLPs, which take no LoRA / DoRA adapter on an MLP Linear "
                             f"(target '{on_mlp[0]}'): disable_fp8 first")
    if getattr(model, "_fp8_proj", False) and not getattr(model, "_fp8_lora", False):
        on_proj = sorted({p[0] for p in plan} & set(model.fp8_proj_linears()))
        if on_proj:
            raise ValueError(f"the model runs FP8 projections, which take no LoRA / DoRA adapter on a projection Linear "
                             f"(target '{on_proj[0]}'): disable_fp8 first")
    extra = sorted(set(weights) - used)
    if extra:
        raise ValueError(f"adapter weights hold {len(extra)} tensors no target uses, e.g. {extra[:3]}")
    with torch.no_grad():
        for name, lin, r, s, A, B, mag in plan:
            wrapped = LoraLinear(lin, r, s, use_dora=mag is not None)
            wrapped.lora_A[ADAPTER].weight.copy_(A)
            wrapped.lora_B[ADAPTER].weight.copy_(B)
            if mag is not None:
                wrapped.lora_magnitude_vector[ADAPTER].weight.copy_(mag)
            parent, _, attr = name.rpartition(".")
            setattr(mods[parent] if parent else model, attr, wrapped)
    _drop_caches(model)
    return model


def unload_lora(model: nn.Module) -> nn.Module:
    """Put the original nn.Linear objects back (the base weights were never modified)."""
    for name, m in list(model.named_modules()):
        if is_wrapped(m):
            parent, _, attr = name.rpartition(".")
            setattr(model.get_submodule(parent) if parent else model, attr, m.base_layer)
    _drop_caches(model)
    return model


def _drop_caches(model: nn.Module) -> None:
    model._drop_caches()
    for m in model.modules():
        proc = getattr(m, "processor", None)
        if proc is not None and hasattr(proc, "_cache"):
            proc._cache.pop(m, None)
