"""LoRA adapters for MMDiT inference, kept unmerged as the reference keeps them (`PeftModel.from_pretrained(model, path,
is_trainable=False)`, opensora/utils/sampling.py:542-545).

`load_lora(model, path, adapter_name=...)` reads a PEFT adapter directory (adapter_config.json +
adapter_model.safetensors / .bin) and replaces every targeted `nn.Linear` with a `LoraLinear`, which has the attribute
layout of peft's `lora.Linear` (`base_layer`, `lora_A` / `lora_B` ModuleDicts keyed by adapter name, `scaling[name]`,
`active_adapters`, `weight` / `bias` of the base layer).  The MMDiT processors read any Linear through `adapters_of`, so
a model wrapped by peft itself takes the same path.  The forward computes x W^T + (x A^T)(s B)^T in one fp32
accumulator (osb_gemm_lora): merging s B A into the bf16 weight instead would round most of a small update away, and
switching or removing an adapter would rewrite the base weights.

Restated from peft's LoraConfig semantics (peft is not a dependency): `target_modules` as a list matches a module whose
name equals an entry or ends with "." + entry, as a string it is a regex full match; `rank_pattern` / `alpha_pattern`
keys match a module name that ends with the pattern (regex) at a "." boundary; scaling = lora_alpha / r, or
lora_alpha / sqrt(r) with `use_rslora`, times `scale`.  `lora_dropout` is inference-irrelevant and ignored.

DoRA (`use_dora`, weight-decomposed LoRA): peft's forward is base(x) + (g - 1) x W^T + g s x A^T B^T with
g = m / ||W + s B A||_2 per output row (m = `lora_magnitude_vector`), i.e. g * (x W^T + s x A^T B^T) + bias.  g is
computed once per pack, in fp32 on the weights' device, and the kernel multiplies its accumulator by it before the bias
(osb_lora_args.col_scale).

Several adapters (`load_lora` under several names, `set_adapters(model, names, weights)`): peft applies the active
adapters of a Linear in order to one running result (`_stack_factors`), each with s = scaling * the user's weight.
That unrolls to one accumulator, so a stack runs on the same packs and launches as one adapter of the summed rank.
Everything else an adapter could ask for (trained biases, modules_to_save, layer selection, fan_in_fan_out) is
refused."""
from __future__ import annotations

import json
import math
import os
import re
import weakref
from typing import NamedTuple

import torch
from torch import Tensor, nn

ADAPTER = "default"


class Adapter(NamedTuple):
    """One active adapter of a Linear as the forward reads it.  `scaling` is the effective s: the layer's scaling times
    the user's weight (`set_adapters`).  `magnitude` is DoRA's m [out_features], None for plain LoRA."""
    name: str
    A: Tensor
    B: Tensor
    scaling: float
    magnitude: Tensor | None


class DoraMagnitude(nn.Module):
    """peft's `DoraLinearLayer` as far as inference reads it: the magnitude vector m [out_features] as `.weight`."""

    def __init__(self, out_features: int, device=None, dtype=None):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(out_features, device=device, dtype=dtype))


class LoraLinear(nn.Module):
    """An `nn.Linear` with unmerged low-rank adapters in peft's `lora.Linear` attribute layout: per adapter name
    `lora_A[name]`, `lora_B[name]`, `scaling[name]`, `use_dora[name]` and, for DoRA, `lora_magnitude_vector[name].weight`;
    `active_adapters` lists the adapters the forward applies, in order.  `adapter_weight[name]` is the user's weight
    (`set_adapters`); peft folds it into `scaling` instead (`set_scale`)."""

    def __init__(self, base: nn.Linear, r: int, scaling: float, use_dora: bool = False, adapter_name: str = ADAPTER):
        super().__init__()
        self.base_layer = base
        self.lora_A, self.lora_B, self.lora_magnitude_vector = nn.ModuleDict(), nn.ModuleDict(), nn.ModuleDict()
        self.scaling, self.use_dora, self.adapter_weight = {}, {}, {}
        self.in_features, self.out_features = base.in_features, base.out_features
        self.add_adapter(adapter_name, r, scaling, use_dora)
        self.active_adapters = [adapter_name]

    def add_adapter(self, name: str, r: int, scaling: float, use_dora: bool = False) -> None:
        """Adapter `name` with rank r and weight 1; it is not made active."""
        w = self.base_layer.weight
        kw = dict(bias=False, device=w.device, dtype=w.dtype)
        self.lora_A[name] = nn.Linear(self.in_features, r, **kw)
        self.lora_B[name] = nn.Linear(r, self.out_features, **kw)
        self.scaling[name], self.use_dora[name], self.adapter_weight[name] = float(scaling), bool(use_dora), 1.0
        if use_dora:
            self.lora_magnitude_vector[name] = DoraMagnitude(self.out_features, w.device, w.dtype)

    def remove_adapter(self, name: str) -> None:
        for d in (self.lora_A, self.lora_B, self.lora_magnitude_vector, self.scaling, self.use_dora, self.adapter_weight):
            if name in d:
                del d[name]
        self.active_adapters = [n for n in self.active_adapters if n != name]

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
        return ", ".join(f"{n}(r={self.lora_A[n].out_features}, scaling={self.scaling[n]}"
                         f"{', use_dora=True' if self.use_dora[n] else ''})" for n in self.lora_A)


def is_wrapped(module: nn.Module) -> bool:
    """True for a LoRA-wrapped Linear, this module's or peft's."""
    return hasattr(module, "base_layer") and hasattr(module, "lora_A")


def adapters_of(lin: nn.Module) -> list[Adapter]:
    """The active adapters of a Linear in the order its forward applies them: peft's `active_adapters`, skipping names the
    layer does not hold.  [] for a plain Linear, and for a peft layer whose adapters are disabled or merged into the base
    weight."""
    la = getattr(lin, "lora_A", None)
    if la is None or getattr(lin, "merged", False) or getattr(lin, "disable_adapters", False):
        return []
    weights, dora = getattr(lin, "adapter_weight", {}), getattr(lin, "use_dora", {})
    return [Adapter(n, la[n].weight, lin.lora_B[n].weight, float(lin.scaling[n]) * weights.get(n, 1.0),
                    lin.lora_magnitude_vector[n].weight if dora.get(n, False) else None)
            for n in getattr(lin, "active_adapters", list(la.keys())) if n in la]


def _single(lin: nn.Module):
    ads = adapters_of(lin)
    if len(ads) > 1:
        raise NotImplementedError(f"{len(ads)} active LoRA adapters on one Linear: adapter_of reads one, adapters_of "
                                  "reads them all")
    return ads[0] if ads else None


def adapter_of(lin: nn.Module):
    """(A [r, in], B [out, r], scaling) of the one active adapter of a LoRA-wrapped Linear, or None for a plain Linear
    (and for a peft layer whose adapters are disabled or already merged into the base weight).  A DoRA adapter also has
    a magnitude vector: `dora_magnitude`.  Several active adapters raise: `adapters_of` reads a stack."""
    ad = _single(lin)
    return None if ad is None else (ad.A, ad.B, ad.scaling)


def dora_magnitude(lin: nn.Module):
    """The magnitude vector m [out_features] of the one active adapter when it is a DoRA adapter, else None."""
    ad = _single(lin)
    return None if ad is None else ad.magnitude


def _state(lins):
    """What a packed adapter depends on: per Linear, the name, order and effective scaling of every active adapter and
    the identity and version of its A / B tensors; for DoRA also of the magnitude vector and the base weight, which
    g = m / ||W + s B A|| reads."""
    out = []
    for lin in lins:
        st = []
        for ad in adapters_of(lin):
            e = (ad.name, ad.A.data_ptr(), ad.A._version, ad.B.data_ptr(), ad.B._version, ad.scaling, ad.A.dtype,
                 ad.A.device)
            if ad.magnitude is not None:
                e += (ad.magnitude.data_ptr(), ad.magnitude._version, lin.weight.data_ptr(), lin.weight._version)
            st.append(e)
        out.append((id(lin), tuple(st)) if st else None)
    return tuple(out)


_PACKS = weakref.WeakKeyDictionary()   # first Linear of a pack -> {layout: (adapter state, pack)}


def lora_pack(groups, k_pad: int = 0):
    """The adapters of Linears that read ONE input, for one down GEMM: `groups` lists, per weight the forward multiplies
    that input with, its output rows as (linear, row_lo, row_hi) slices (a packed q|k|v weight has three; linear1's qkv
    part is (linear1, 0, 3C)).  Returns None when no member has an active adapter, else
    (A_cat, [B_cat or None per group], [col_scale or None per group]): A_cat bf16 [R, K + k_pad] stacks the A of every
    active adapter of every member once (rank zero-padded to a multiple of 8, K zero-padded by k_pad like the base
    weight); B_cat bf16 [rows, R] holds each adapter's c * s * B in its member's rows and its rank columns and zeros
    elsewhere, None for a group without an adapted member; col_scale fp32 [rows] holds G in the rows of a member whose
    stack has a DoRA adapter and 1.0 elsewhere, None for a group without one.  c and G come from `_stack_factors`; for a
    single adapter c = 1 and G = g.  Cached on the adapter state."""
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


def _stack_factors(lin, ads):
    """A stack of adapters k = 1..K applied in order, as peft's `lora.Linear.forward` applies them in eval mode
    (restated, unpinned: DESIGN.md 4.1c): LoRA adds s_k x A_k^T B_k^T to the running result; DoRA multiplies the running
    result (bias excluded) plus its own update by g_k = m_k / ||W + s_k B_k A_k||, so the order matters.  This unrolls
    to one accumulator, G * (x W^T + sum_k c_k s_k x A_k^T B_k^T), with G the product of the g_j of all DoRA adapters
    and c_k = 1 / the product of those before k.  Returns ([c_k s_k per adapter: a float, or fp32 [out] once a DoRA
    adapter came before], G fp32 [out] or None without DoRA)."""
    facs, G = [], None
    for ad in ads:
        facs.append(ad.scaling if G is None else ad.scaling / G)
        if ad.magnitude is not None:
            g = _dora_scale(lin, ad.A, ad.B, ad.scaling, ad.magnitude)
            G = g if G is None else G * g
    return facs, G


def _build_pack(groups, lins, k_pad):
    ads = {id(l): adapters_of(l) for l in lins}
    offs, R = {}, 0   # (Linear, adapter index) -> first row in A_cat
    for lin in lins:
        for k, ad in enumerate(ads[id(lin)]):
            offs[id(lin), k] = R
            R += -(-ad.A.shape[0] // 8) * 8
    ref = next(a for a in ads.values() if a)[0].A
    K = ref.shape[1]
    with torch.no_grad():
        A_cat = torch.zeros(R, K + k_pad, dtype=torch.bfloat16, device=ref.device)
        for lin in lins:
            for k, ad in enumerate(ads[id(lin)]):
                A_cat[offs[id(lin), k]:offs[id(lin), k] + ad.A.shape[0], :K] = ad.A
        fac = {id(l): _stack_factors(l, ads[id(l)]) for l in lins if ads[id(l)]}
        Bs = []
        for g in groups:
            if all(not ads[id(l)] for l, _, _ in g):
                Bs.append(None)
                continue
            Bg = torch.zeros(sum(hi - lo for _, lo, hi in g), R, dtype=torch.float32, device=ref.device)
            row = 0
            for lin, lo, hi in g:
                for k, ad in enumerate(ads[id(lin)]):
                    f, o = fac[id(lin)][0][k], offs[id(lin), k]
                    f = f if isinstance(f, float) else f[lo:hi, None]
                    Bg[row:row + hi - lo, o:o + ad.A.shape[0]] = f * ad.B[lo:hi].float()
                row += hi - lo
            Bs.append(Bg.to(torch.bfloat16).contiguous())   # bf16(c s B): folded once per load / change
        Ss = []
        for g in groups:
            if all(id(l) not in fac or fac[id(l)][1] is None for l, _, _ in g):
                Ss.append(None)
                continue
            Ss.append(torch.cat([fac[id(l)][1][lo:hi] if id(l) in fac and fac[id(l)][1] is not None
                                 else torch.ones(hi - lo, device=ref.device) for l, lo, hi in g]).contiguous())
    return A_cat, Bs, Ss


_NORM_CHUNK = 1 << 24   # fp32 elements of W + s B A materialised at a time while g is computed (64 MB)


def _dora_scale(lin, A, B, s, m=None):
    """g = m / ||W + s B A||_2 over in_features, fp32 [out_features], on the weights' device (m: the magnitude vector,
    by default the one active adapter's); computed in row chunks so the temporary stays bounded whatever the layer's
    size.  (peft's DoRA layer recomputes this on every forward.)"""
    W = lin.weight
    Af = A.float()
    norm = torch.empty(W.shape[0], dtype=torch.float32, device=W.device)
    step = max(1, _NORM_CHUNK // W.shape[1])
    for lo in range(0, W.shape[0], step):
        hi = min(lo + step, W.shape[0])
        norm[lo:hi] = torch.linalg.vector_norm(W[lo:hi].float() + s * (B[lo:hi].float() @ Af), dim=1)
    return (dora_magnitude(lin) if m is None else m).float() / norm


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


def _modules(model: nn.Module) -> list:
    """(name, module) of every module as an adapter config names them: a wrapped Linear under its own name, and nothing
    inside it (its base layer and adapter Linears are not targets)."""
    out = []

    def walk(mod, prefix):
        for n, c in mod.named_children():
            out.append((prefix + n, c))
            if not is_wrapped(c):
                walk(c, prefix + n + ".")

    walk(model, "")
    return out


def _targets(model: nn.Module, target_modules) -> list[str]:
    names = [n for n, _ in _modules(model)]
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


def _wrappers(model: nn.Module) -> list:
    """(name, LoraLinear) of every Linear `load_lora` wrapped."""
    return [(n, m) for n, m in model.named_modules() if isinstance(m, LoraLinear)]


def active_adapters(model: nn.Module) -> list[str]:
    """The names of the model's active adapters, in the order the forward applies them."""
    names = []
    for _, w in _wrappers(model):
        names += [n for n in w.active_adapters if n not in names]
    return names


def _refuse_fp8_targets(model: nn.Module, names) -> None:
    """Adapters on Linears that run on e4m3 need enable_fp8(..., lora=True)."""
    if getattr(model, "_fp8_lora", False):
        return
    if getattr(model, "_fp8", False):
        on_mlp = sorted(set(names) & set(model.fp8_mlp_linears()))
        if on_mlp:
            raise ValueError(f"the model runs FP8 MLPs, which take no LoRA / DoRA adapter on an MLP Linear "
                             f"(target '{on_mlp[0]}'): disable_fp8 first")
    if getattr(model, "_fp8_proj", False):
        on_proj = sorted(set(names) & set(model.fp8_proj_linears()))
        if on_proj:
            raise ValueError(f"the model runs FP8 projections, which take no LoRA / DoRA adapter on a projection Linear "
                             f"(target '{on_proj[0]}'): disable_fp8 first")


def load_lora(model: nn.Module, path: str, scale: float = 1.0, adapter_name: str = ADAPTER) -> nn.Module:
    """Load the PEFT LoRA adapter in directory `path` into the MMDiT `model` as adapter `adapter_name`, in place,
    unmerged; `scale` multiplies every layer's scaling (lora_alpha / r).  A DoRA adapter (`use_dora: true`) also carries
    one magnitude vector per target, saved by peft as `base_model.model.<name>.lora_magnitude_vector` [out_features] (its
    state-dict export drops the adapter name and the DoRA layer's `.weight`).

    Several adapters stack as in peft: a Linear that already carries adapters gets the new one next to them, and the new
    adapter is appended to the active list with weight 1 (`set_adapters` changes both).  A name the model already
    carries is refused.  Returns the model."""
    from opensora.models.mmdit.model import MMDiTModel

    if not isinstance(model, MMDiTModel):
        raise TypeError(f"load_lora supports MMDiTModel only, got {type(model).__name__}")
    for name, m in model.named_modules():
        if is_wrapped(m) and not isinstance(m, LoraLinear):
            raise ValueError(f"the model already carries a LoRA layer of another package (at '{name}'): unload_lora first")
        if isinstance(m, LoraLinear) and adapter_name in m.lora_A:
            raise ValueError(f"the model already carries a LoRA adapter named {adapter_name!r} (at '{name}'): "
                             "unload_lora first, or load it under another adapter_name")
    cfg = _read_config(path)
    weights = _read_weights(path)
    prefix = "base_model.model."
    r0, alpha0 = int(cfg.get("r", 8)), float(cfg.get("lora_alpha", 8))
    dora = bool(cfg.get("use_dora"))
    mods = dict(_modules(model))
    plan, used = [], set()
    for name in _targets(model, cfg["target_modules"]):
        lin = mods[name]
        if type(lin) is not nn.Linear and not isinstance(lin, LoraLinear):
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
    _refuse_fp8_targets(model, [p[0] for p in plan])
    extra = sorted(set(weights) - used)
    if extra:
        raise ValueError(f"adapter weights hold {len(extra)} tensors no target uses, e.g. {extra[:3]}")
    active = active_adapters(model) + [adapter_name]
    with torch.no_grad():
        for name, lin, r, s, A, B, mag in plan:
            if isinstance(lin, LoraLinear):
                wrapped = lin
                wrapped.add_adapter(adapter_name, r, s, use_dora=mag is not None)
            else:
                wrapped = LoraLinear(lin, r, s, use_dora=mag is not None, adapter_name=adapter_name)
                parent, _, attr = name.rpartition(".")
                setattr(mods[parent] if parent else model, attr, wrapped)
            wrapped.lora_A[adapter_name].weight.copy_(A)
            wrapped.lora_B[adapter_name].weight.copy_(B)
            if mag is not None:
                wrapped.lora_magnitude_vector[adapter_name].weight.copy_(mag)
    for _, w in _wrappers(model):
        w.active_adapters = list(active)
    _drop_caches(model)
    return model


def set_adapters(model: nn.Module, names, weights=None) -> nn.Module:
    """Make `names` the model's active adapters, applied in that order, with one weight each (default 1.0).  A weight w
    multiplies the adapter's scaling s wherever the forward reads s, in DoRA's norm ||W + s B A|| too, as peft's
    `set_scale` does.  [] runs the base model.  Names that are not loaded, or repeated, are refused.  Returns the
    model."""
    names = [names] if isinstance(names, str) else list(names)
    weights = [1.0] * len(names) if weights is None else [float(w) for w in weights]
    if len(weights) != len(names):
        raise ValueError(f"set_adapters: {len(names)} adapters but {len(weights)} weights")
    if len(set(names)) != len(names):
        raise ValueError(f"set_adapters: an adapter is named twice in {names}")
    wraps = _wrappers(model)
    loaded = {n for _, w in wraps for n in w.lora_A}
    unknown = [n for n in names if n not in loaded]
    if unknown:
        raise ValueError(f"set_adapters: no adapter named {unknown[0]!r} is loaded (loaded: {sorted(loaded)})")
    _refuse_fp8_targets(model, [n for n, w in wraps if any(a in w.lora_A for a in names)])
    for _, w in wraps:
        w.active_adapters = list(names)
        for n, x in zip(names, weights):
            if n in w.lora_A:
                w.adapter_weight[n] = x
    _drop_caches(model)
    return model


def unload_lora(model: nn.Module, adapter_name: str | None = None) -> nn.Module:
    """Remove adapter `adapter_name` (None: every adapter) and put back the original nn.Linear of every Linear left
    without one (the base weights were never modified).  Returns the model."""
    if adapter_name is None:
        for name, m in list(model.named_modules()):
            if is_wrapped(m):
                parent, _, attr = name.rpartition(".")
                setattr(model.get_submodule(parent) if parent else model, attr, m.base_layer)
    else:
        wraps = _wrappers(model)
        if not any(adapter_name in w.lora_A for _, w in wraps):
            raise ValueError(f"unload_lora: no adapter named {adapter_name!r} is loaded")
        for name, w in wraps:
            w.remove_adapter(adapter_name)
            if not len(w.lora_A):
                parent, _, attr = name.rpartition(".")
                setattr(model.get_submodule(parent) if parent else model, attr, w.base_layer)
    _drop_caches(model)
    return model


def _drop_caches(model: nn.Module) -> None:
    model._drop_caches()
    for m in model.modules():
        proc = getattr(m, "processor", None)
        if proc is not None and hasattr(proc, "_cache"):
            proc._cache.pop(m, None)
