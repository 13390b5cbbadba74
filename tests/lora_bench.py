"""Measurement of LoRA inference on one GPU; prints one JSON line.

  python tests/lora_bench.py [--reps 5] [--iters 10] [--no-model]

- The MMDiT GEMMs at the 256px inference shape (M = 3 x (8316 + 512) = 26 484 token rows, C = 3072): qkv 3072 -> 9216,
  proj 3072 -> 3072, MLP 3072 -> 12288 -> 3072, linear1 3072 -> 21504, linear2 15360 -> 3072.  For r in {16, 64, 128}:
  osb_gemm_bf16 alone against the adapted pair (down GEMM U = x A^T, then osb_gemm_lora), alternated, median of --reps
  windows of --iters calls each; the two parts of the pair are also timed on their own.
- The whole MMDiT 256px forward (bench.py's mmdit leg: B = 3, random bf16 weights created on the device) with no adapter
  and with an r = 64 adapter on every block Linear, alternated, median.
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
            u = osb200.gemm(x, A)
            t = alternate({
                "base": lambda: osb200.gemm(x, w, b, out=out),
                "adapted": lambda: osb200.gemm_lora(x, w, b, osb200.gemm(x, A), Bm, out=out),
                "down": lambda: osb200.gemm(x, A, out=u),
                "fused": lambda: osb200.gemm_lora(x, w, b, u, Bm, out=out),
            }, reps, iters)
            t["overhead_pct"] = round(100.0 * (t["adapted"] / t["base"] - 1.0), 2)
            t["base_tflops"] = round(2.0 * M_ROWS * N * K / (t["base"] * 1e-3) / 1e12, 1)
            res[f"{name}_r{r}"] = t
    return res


def model(reps):
    import osb200
    from opensora.utils.lora import LoraLinear

    plain, inp = mmdit_256px()
    res = {}
    with torch.no_grad():
        out_plain = plain(**inp).clone()
        l0 = osb200.launch_count()
        plain(**inp)
        res["launches_plain"] = osb200.launch_count() - l0
        # r = 64 on every Linear of every block (the same model object: the adapter is put on and taken off in place)
        wrapped = []
        for blocks in (plain.double_blocks, plain.single_blocks):
            for name, m in list(blocks.named_modules()):
                if type(m) is torch.nn.Linear:
                    parent, _, attr = name.rpartition(".")
                    lin = LoraLinear(m, 64, 1.0)
                    torch.nn.init.normal_(lin.lora_A["default"].weight, std=m.in_features ** -0.5)
                    torch.nn.init.normal_(lin.lora_B["default"].weight, std=1e-3)
                    wrapped.append((blocks.get_submodule(parent) if parent else blocks, attr, m, lin))
        res["adapted_linears"] = len(wrapped)

        def put(on: bool):
            for parent, attr, m, lin in wrapped:
                setattr(parent, attr, lin if on else m)
            plain._drop_caches()

        put(True)
        out_lora = plain(**inp)
        l0 = osb200.launch_count()
        plain(**inp)
        res["launches_lora"] = osb200.launch_count() - l0
        res["finite"] = bool(torch.isfinite(out_lora.float()).all())
        res["rel_change"] = float((out_lora.float() - out_plain.float()).norm() / out_plain.float().norm())
        t = {"plain": [], "lora": []}
        for _ in range(reps):
            for k in ("plain", "lora"):
                put(k == "lora")
                plain(**inp)   # repacks after the swap (off the clock)
                t[k].append(window_ms(lambda: plain(**inp), 1))
        put(False)
    res.update({f"{k}_ms": round(statistics.median(v), 2) for k, v in t.items()})
    res.update({f"{k}_spread_ms": round(max(v) - min(v), 2) for k, v in t.items()})
    res["overhead_pct"] = round(100.0 * (res["lora_ms"] / res["plain_ms"] - 1.0), 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
    import osb200

    osb200.init(0)
    name, power = card()
    res = {"card": name, "power_limit,max_sm_clock": power, "rows": M_ROWS, "gemm_ms": gemms(a.reps, a.iters)}
    if not a.no_model:
        res["mmdit_256px_forward"] = model(a.reps)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
