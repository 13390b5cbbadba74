"""Measurement of DoRA inference on one GPU; prints one JSON line.

  python tests/dora_bench.py [--reps 5] [--iters 10] [--no-model]

- At the MMDiT GEMM shapes of the 256px inference step (tests/lora_bench.py: M = 26 484 token rows), for r in
  {16, 64, 128}: osb_gemm_lora without and with `col_scale` (same U and s B, alternated), the whole adapted pair (down GEMM
  + osb_gemm_lora with col_scale), and a peft-style eager DoRA layer on the same operands (torch: base GEMM, the two LoRA
  GEMMs, s B A and its row norm on every call, as peft's DoraLinearLayer does).  Median of --reps windows of --iters calls.
- The whole MMDiT 256px forward (bench.py's mmdit leg: B = 3) with no adapter, with an r = 64 LoRA adapter and with an
  r = 64 DoRA adapter on every block Linear, alternated, median.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-sora_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tests.models import GEMMS_256PX as SHAPES, ROWS_256PX as M_ROWS, mmdit_256px  # noqa: E402
from tests.timing import alternate, card, window_ms  # noqa: E402


def _peft_dora(x, w, b, A, B, s, m):
    """peft's DoraLinearLayer.forward at inference, with the base result passed in (one base GEMM)."""
    base = torch.nn.functional.linear(x, w, b)
    lora = torch.nn.functional.linear(torch.nn.functional.linear(x, A), B)
    weight_norm = torch.linalg.norm(w + s * (B @ A), dim=1).to(w.dtype)
    g = (m / weight_norm).view(1, -1)
    return base + (g - 1) * (base - b) + g * lora * s


def gemms(reps, iters):
    import osb200

    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).to(torch.bfloat16)   # noqa: E731
    res = {}
    for name, (K, N) in SHAPES.items():
        x, w, b = rn(M_ROWS, K), rn(N, K, sc=K ** -0.5), rn(N, sc=0.1)
        out = torch.empty(M_ROWS, N, dtype=torch.bfloat16, device="cuda")
        for r in (16, 64, 128):
            A, Bm = rn(r, K, sc=K ** -0.5), rn(N, r, sc=0.01)
            m = (w.float().norm(dim=1) * 1.1).to(torch.bfloat16)
            cs = torch.rand(N, device="cuda", generator=g) + 0.5
            u = osb200.gemm(x, A)
            t = alternate({
                "fused_lora": lambda: osb200.gemm_lora(x, w, b, u, Bm, out=out),
                "fused_dora": lambda: osb200.gemm_lora(x, w, b, u, Bm, out=out, col_scale=cs),
                "dora_pair": lambda: osb200.gemm_lora(x, w, b, osb200.gemm(x, A), Bm, out=out, col_scale=cs),
                "peft_eager_dora": lambda: _peft_dora(x, w, b, A, Bm, 1.0, m),
            }, reps, iters)
            t["col_scale_pct"] = round(100.0 * (t["fused_dora"] / t["fused_lora"] - 1.0), 2)
            t["eager_over_pair"] = round(t["peft_eager_dora"] / t["dora_pair"], 2)
            res[f"{name}_r{r}"] = t
    return res


def model(reps):
    import osb200
    from opensora.utils.lora import LoraLinear

    net, inp = mmdit_256px()
    res = {}
    with torch.no_grad():
        # r = 64 on every Linear of every block, as LoRA and as DoRA with the same A and B (magnitudes 1.1 x the row
        # norms of W, so g is about 1.1); the adapters are put on and taken off the same model object
        wrapped = []
        for blocks in (net.double_blocks, net.single_blocks):
            for name, lin in list(blocks.named_modules()):
                if type(lin) is torch.nn.Linear:
                    parent, _, attr = name.rpartition(".")
                    lo, do = LoraLinear(lin, 64, 1.0), LoraLinear(lin, 64, 1.0, use_dora=True)
                    torch.nn.init.normal_(lo.lora_A["default"].weight, std=lin.in_features ** -0.5)
                    torch.nn.init.normal_(lo.lora_B["default"].weight, std=1e-3)
                    do.lora_A, do.lora_B = lo.lora_A, lo.lora_B
                    do.lora_magnitude_vector["default"].weight.copy_(lin.weight.float().norm(dim=1) * 1.1)
                    wrapped.append((blocks.get_submodule(parent) if parent else blocks, attr, lin, lo, do))
        res["adapted_linears"] = len(wrapped)

        def put(kind: str):
            for parent, attr, lin, lo, do in wrapped:
                setattr(parent, attr, {"plain": lin, "lora": lo, "dora": do}[kind])
            net._drop_caches()

        outs = {}
        for k in ("plain", "lora", "dora"):
            put(k)
            outs[k] = net(**inp).float()   # builds the packs (and g) off the clock
            l0 = osb200.launch_count()
            net(**inp)
            res[f"launches_{k}"] = osb200.launch_count() - l0
        res["finite"] = all(bool(torch.isfinite(o).all()) for o in outs.values())
        res["dora_vs_lora_rel_change"] = float((outs["dora"] - outs["lora"]).norm() / outs["lora"].norm())
        t = {"plain": [], "lora": [], "dora": []}
        for _ in range(reps):
            for k in t:
                put(k)
                net(**inp)   # re-reads the cached packs after the swap (off the clock)
                t[k].append(window_ms(lambda: net(**inp), 1))
        put("plain")
    res.update({f"{k}_ms": round(statistics.median(v), 2) for k, v in t.items()})
    res.update({f"{k}_spread_ms": round(max(v) - min(v), 2) for k, v in t.items()})
    res["lora_overhead_pct"] = round(100.0 * (res["lora_ms"] / res["plain_ms"] - 1.0), 2)
    res["dora_overhead_pct"] = round(100.0 * (res["dora_ms"] / res["plain_ms"] - 1.0), 2)
    res["dora_over_lora_pct"] = round(100.0 * (res["dora_ms"] / res["lora_ms"] - 1.0), 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dora_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
    import osb200

    osb200.init(0)
    name, power = card()
    res = {"card": name, "power_limit,max_sm_clock": power, "rows": M_ROWS, "gemm_ms": gemms(a.reps, a.iters)}
    if not a.no_model:
        res["mmdit_256px_forward"] = model(a.reps)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
