"""Parity metrics shared by the tests (max-abs, rel-L2 against an fp32 reference)."""
import torch


def rel_l2(a: torch.Tensor, ref: torch.Tensor) -> float:
    a = a.double().flatten()
    ref = ref.double().flatten()
    return float((a - ref).norm() / ref.norm().clamp_min(1e-30))


def max_abs(a: torch.Tensor, ref: torch.Tensor) -> float:
    return float((a.double() - ref.double()).abs().max())


def report(name: str, a: torch.Tensor, ref: torch.Tensor) -> tuple[float, float]:
    r, m = rel_l2(a, ref), max_abs(a, ref)
    print(f"[parity] {name}: rel_l2={r:.3e} max_abs={m:.3e} ref_absmax={float(ref.abs().max()):.3e}")
    return r, m


# one bf16 rounding of an exact result has RMS relative error 2^-9/sqrt(3) ~ 1.1e-3
BF16_ONE_ROUNDING_REL_L2 = 2.0e-3


# ---- golden fixtures (tests/golden/*.npz) -----------------------------------------------------------------------------
# Random weights are not stored: a generator sets every parameter from a seed derived from its name (seeded_init) and
# the fixture keeps the name -> (seed key, parameter name, shape) manifest; load_golden regenerates the same values.
import json as _json  # noqa: E402
import os as _os  # noqa: E402
import zlib as _zlib  # noqa: E402

import numpy as _np  # noqa: E402

GOLDEN = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "golden")
_SEEDED: dict = {}


def seeded_param(key: str, name: str, shape) -> torch.Tensor:
    """Deterministic fp32 value of parameter `name` under seed key `key`: norm weights / scales 1 + 0.2 N(0,1), other
    vectors 0.1 N(0,1), matrices and kernels U(-1, 1) / sqrt(fan_in) (the spread of torch's default Linear / Conv init)."""
    shape = tuple(int(s) for s in shape)
    g = torch.Generator().manual_seed(_zlib.crc32(key.encode()))
    leaf = name.rsplit(".", 1)[-1]
    if len(shape) == 1:
        x = torch.randn(shape, generator=g)
        return 1.0 + 0.2 * x if (leaf == "scale" or (leaf == "weight" and "norm" in name)) else 0.1 * x
    x = torch.rand(shape, generator=g) * 2.0 - 1.0
    return x * (x.numel() // shape[0]) ** -0.5


def seeded_init(module, prefix: str) -> None:
    """Golden generators: overwrite every parameter of `module` with seeded_param(prefix.name)."""
    with torch.no_grad():
        for n, p in module.named_parameters():
            p.copy_(seeded_param(f"{prefix}.{n}", n, p.shape))
            _SEEDED[p.data_ptr()] = (f"{prefix}.{n}", n)


def save_golden(path: str, out: dict, half=()) -> None:
    """Write `out` to `path`: seeded parameters as manifest entries, keys in `half` as float16, the rest as float32."""
    arrays, params = {}, {}
    for k, t in out.items():
        t = t.detach()
        seeded = _SEEDED.get(t.data_ptr()) if t.numel() else None
        if seeded is not None:
            params[k] = [seeded[0], seeded[1], list(t.shape)]
        else:
            arrays[k] = t.float().numpy().astype(_np.float16 if k in half else _np.float32)
    arrays["__seeded_params__"] = _np.array(_json.dumps(params, sort_keys=True))
    _np.savez_compressed(path, **arrays)


def load_golden(name: str) -> dict:
    """tests/golden/<name> as {key: fp32 tensor}, seeded parameters regenerated."""
    z = _np.load(_os.path.join(GOLDEN, name))
    G = {k: torch.from_numpy(z[k].astype(_np.float32)) for k in z.files if k != "__seeded_params__"}
    if "__seeded_params__" in z.files:
        for k, (key, n, shape) in _json.loads(str(z["__seeded_params__"])).items():
            G[k] = seeded_param(key, n, shape)
    return G
