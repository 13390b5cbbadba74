"""Measurement of LoRA adapters on the MMDiT FP8 GEMMs on one GPU; prints one JSON line.

  python tests/mmdit_fp8_lora_bench.py [--reps 5] [--iters 3] [--no-model]

1. Per GEMM at M = 26 484 rows (B = 3 x L = 8 828, C = 3072), r in {16, 64, 128}, alternated windows, medians and
   spreads: the FP8 GEMM alone; the FP8 down GEMM plus osb_gemm_fp8_lora; and the bf16 pair (osb_gemm_bf16 down GEMM plus
   osb_gemm_lora) for comparison.  qkv (3072 -> 9216, per-row A), proj (3072 -> 3072, block A, gate + residual), fc1
   (3072 -> 12288, FP8 GELU epilogue), fc2 (12288 -> 3072, block A, gate + residual), linear1 (its qkv and mlp parts on
   one down GEMM) and linear2 (15360 -> 3072, block A, gate + residual).
2. The whole 256px forward (bench.py's mmdit leg, 19 + 38 blocks) with an r = 64 adapter on every block Linear, alternated,
   median: bf16 GEMMs + LoRA + FP8 attention; FP8 GEMMs (MLPs and projections) + LoRA + FP8 attention; FP8 GEMMs + FP8
   attention with no adapter.  The rel-L2 between the two adapted outputs.
The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-sora_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tests.models import B_256PX as B, L_256PX as L, mmdit_256px  # noqa: E402
from tests.timing import alternate, card, window_ms  # noqa: E402

C = 3072


def ops(reps, iters):
    import osb200

    g = torch.Generator(device="cuda").manual_seed(0)
    M = B * L
    rb = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).to(torch.bfloat16)   # noqa: E731
    GATE = dict(epilogue=osb200.EPI_BIAS_GATE_RES, gate=torch.randn(1, C, device="cuda", generator=g))
    # name: (K, [(N, bf16 epilogue, fp8 epilogue)] parts reading one input, block-scaled A)
    gemms = {"qkv": (C, [(3 * C, osb200.EPI_BIAS, osb200.EPI_BIAS)], False),
             "proj": (C, [(C, "gate", "gate")], True),
             "fc1": (C, [(4 * C, osb200.EPI_BIAS_GELU_TANH, osb200.EPI_BIAS_GELU_TANH_FP8)], False),
             "fc2": (4 * C, [(C, "gate", "gate")], True),
             "linear1": (C, [(3 * C, osb200.EPI_BIAS, osb200.EPI_BIAS),
                             (4 * C, osb200.EPI_BIAS_GELU_TANH, osb200.EPI_BIAS_GELU_TANH_FP8)], False),
             "linear2": (5 * C, [(C, "gate", "gate")], True)}
    res = {}
    for name, (K, parts, block_a) in gemms.items():
        x = rb(M, K)
        x8, xs = osb200.quant_blocks_fp8(x) if block_a else osb200.quant_rows_fp8(x)
        res_x = rb(M, C)
        ps = []
        for N, e16, e8 in parts:
            w = rb(N, K, sc=K ** -0.5)
            w8, ws = osb200.quant_blocks_fp8(w, block=K)
            kw16 = dict(GATE, residual=res_x, out=res_x) if e16 == "gate" else dict(epilogue=e16)
            kw8 = dict(GATE, residual=res_x, out=res_x) if e8 == "gate" else dict(epilogue=e8)
            ps.append((N, w, rb(N, sc=0.02), w8, ws.view(-1), kw16, kw8))
        for r in (16, 64, 128):
            A = rb(r, K, sc=K ** -0.5)
            A8, As = osb200.quant_blocks_fp8(A, block=K)
            Bs = [rb(N, r, sc=0.1 * r ** -0.5) for N, *_ in ps]

            def fp8():
                for N, w, bias, w8, ws, kw16, kw8 in ps:
                    osb200.gemm_fp8_blocks(x8, xs, w8, ws, bias, **kw8)

            def fp8_lora():
                u = osb200.gemm_fp8_blocks(x8, xs, A8, As.view(-1))
                for (N, w, bias, w8, ws, kw16, kw8), Bm in zip(ps, Bs):
                    osb200.gemm_fp8_lora(x8, xs, w8, ws, bias, u, Bm, **kw8)

            def bf16_lora():
                u = osb200.gemm(x, A)
                for (N, w, bias, w8, ws, kw16, kw8), Bm in zip(ps, Bs):
                    osb200.gemm_lora(x, w, bias, u, Bm, **kw16)

            t = alternate({"fp8": fp8, "fp8_down_plus_fp8_lora": fp8_lora, "bf16_down_plus_bf16_lora": bf16_lora},
                           reps, iters)
            t["fp8_lora_over_fp8"] = round(t["fp8_down_plus_fp8_lora"] / t["fp8"], 3)
            t["fp8_lora_speedup_over_bf16_lora"] = round(t["bf16_down_plus_bf16_lora"] / t["fp8_down_plus_fp8_lora"], 3)
            res[f"{name}_M{M}_K{K}_N{'+'.join(str(p[0]) for p in ps)}_r{r}"] = t
    return res


def model(net, inp, reps):
    from opensora.utils.lora import load_lora, unload_lora
    from tests.adapters import write_adapter

    targets = net.fp8_mlp_linears() + net.fp8_proj_linears()
    tmp = tempfile.mkdtemp()
    path = write_adapter(os.path.join(tmp, "a"), net, r=64, alpha=64, rel=0.1, seed=1, targets=targets)
    net.enable_fp8_attention()
    modes = ("bf16_lora_fp8_attention", "fp8_lora_fp8_attention", "fp8_no_adapter_fp8_attention")

    def setmode(m):
        adapted = any(hasattr(mod, "lora_A") for mod in net.modules())
        if m == "fp8_no_adapter_fp8_attention":
            if adapted:
                unload_lora(net)
            net.enable_fp8(projections=True)
            return
        net.disable_fp8()   # the default FP8 path refuses adapters: load with FP8 off
        if not adapted:
            load_lora(net, path)
        if m == "fp8_lora_fp8_attention":
            net.enable_fp8(projections=True, lora=True)

    res, outs = {}, {}
    t = {m: [] for m in modes}
    with torch.no_grad():
        for m in modes:
            setmode(m)
            outs[m] = net(**inp).float()
        a, b = outs["fp8_lora_fp8_attention"], outs["bf16_lora_fp8_attention"]
        res["fp8_lora_vs_bf16_lora_rel_l2"] = float((a - b).norm() / b.norm())
        for i in range(reps):
            for m in (list(modes) if i % 2 == 0 else list(modes)[::-1]):
                setmode(m)
                net(**inp)   # quantizes the weights / warms the workspaces off the clock
                t[m].append(window_ms(lambda: net(**inp), 1))
    res.update({f"{m}_ms": round(statistics.median(v), 2) for m, v in t.items()})
    res.update({f"{m}_spread_ms": round(max(v) - min(v), 2) for m, v in t.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mmdit_fp8_lora_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
    import osb200

    osb200.init(0)
    name, power = card()
    res = {"card": name, "power_limit,max_sm_clock": power, "ops": ops(a.reps, a.iters)}
    if not a.no_model:
        net, inp = mmdit_256px()
        res["mmdit_256px_forward"] = model(net, inp, a.reps)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
