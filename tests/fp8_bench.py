"""FP8 (e4m3) MLPs against bf16 on one GPU: the two MLP GEMMs of STDiT3-XL/2 at M = 16 384 tokens (the fc2 input
quantizer timed on its own), and the whole XL/2 denoising step (1x4x64x32x32) with FP8 MLPs against bf16, eager and as
a CUDA graph.  Each figure is the median of 5 windows of at least 200 ms of work each (the call count per window is
calibrated per variant), the variants alternating window by window.  Prints the card, its power limit and its max SM
clock from the same run.

    python tests/fp8_bench.py [--steps 5]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "open-sora_b200")]

from tests.timing import card, window_ms  # noqa: E402


def alternate(fns: dict, min_iters: int, windows: int = 5, window_ms_min: float = 200.0):
    iters = {}
    for k, f in fns.items():   # warm-up (module load, descriptors, allocator), then size the window
        window_ms(f, 2)
        iters[k] = max(min_iters, int(window_ms_min / window_ms(f, min_iters)) + 1)
    t = {k: [] for k in fns}
    for _ in range(windows):
        for k, f in fns.items():
            t[k].append(window_ms(f, iters[k]))
    return {k: statistics.median(v) for k, v in t.items()}


def gemms():
    import osb200

    M, C = 16384, 1152
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(M, C, device="cuda", generator=g).to(torch.bfloat16)
    h = torch.randn(M, 4 * C, device="cuda", generator=g).to(torch.bfloat16)
    w1 = (torch.randn(4 * C, C, device="cuda", generator=g) / C ** 0.5).to(torch.bfloat16)
    w2 = (torch.randn(C, 4 * C, device="cuda", generator=g) / (4 * C) ** 0.5).to(torch.bfloat16)
    b1 = torch.zeros(4 * C, device="cuda", dtype=torch.bfloat16)
    b2 = torch.zeros(C, device="cuda", dtype=torch.bfloat16)
    gate = torch.ones(1, C, device="cuda")
    x8, xs = osb200.quant_rows_fp8(x)
    w18, w1s = osb200.quant_rows_fp8(w1)
    w28, w2s = osb200.quant_rows_fp8(w2)
    h8, hs = osb200.quant_rows_fp8(h)
    o1 = torch.empty(M, 4 * C, device="cuda", dtype=torch.bfloat16)
    o2 = torch.empty(M, C, device="cuda", dtype=torch.bfloat16)
    G1, G2 = osb200.EPI_BIAS_GELU_TANH, osb200.EPI_BIAS_GATE_RES
    fns = {
        "fc1_bf16": lambda: osb200.gemm(x, w1, b1, epilogue=G1, out=o1),
        "fc1_fp8": lambda: osb200.gemm_fp8(x8, xs, w18, w1s, b1, epilogue=G1, out=o1),
        "fc2_bf16": lambda: osb200.gemm(h, w2, b2, epilogue=G2, residual=o2, gate=gate, out=o2),
        "fc2_fp8": lambda: osb200.gemm_fp8(h8, hs, w28, w2s, b2, epilogue=G2, residual=o2, gate=gate, out=o2),
        "quant_fc2_input": lambda: osb200.quant_rows_fp8(h, out=h8, out_scale=hs),
    }
    t = alternate(fns, 20)
    flops = 2.0 * M * 4 * C * C
    res = {k: {"ms": round(v, 4)} for k, v in t.items()}
    for k in ("fc1_bf16", "fc1_fp8", "fc2_bf16", "fc2_fp8"):
        res[k]["tflops"] = round(flops / t[k] / 1e9, 1)
    res["quant_fc2_input"]["gb_per_s"] = round(3.0 * M * 4 * C / t["quant_fc2_input"] / 1e6, 1)
    res["mlp_speedup_incl_quant"] = round((t["fc1_bf16"] + t["fc2_bf16"]) /
                                          (t["fc1_fp8"] + t["fc2_fp8"] + t["quant_fc2_input"]), 3)
    return res


def step(steps: int):
    from tests.models import stdit3_inputs, stdit3_pair

    bf, _, cfg = stdit3_pair("xl")
    f8, _, _ = stdit3_pair("xl")
    f8.enable_fp8()
    inp = stdit3_inputs(cfg, 1, 64, 32, 32, lens=[260], device="cuda")
    with torch.no_grad():
        fns = {"step_bf16_eager": lambda: bf(**inp), "step_fp8_eager": lambda: f8(**inp)}
        t = alternate(fns, steps)
        gb, g8 = bf.capture(**inp), f8.capture(**inp)
        t.update(alternate({"step_bf16_graph": lambda: gb(**inp), "step_fp8_graph": lambda: g8(**inp)}, steps))
    res = {k: round(v, 2) for k, v in t.items()}
    res["speedup_eager"] = round(t["step_bf16_eager"] / t["step_fp8_eager"], 3)
    res["speedup_graph"] = round(t["step_bf16_graph"] / t["step_fp8_graph"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py measures on a CUDA device; there is none")
    import osb200

    osb200.init()
    out = {"card": ", ".join(card()), "mlp_gemms_m16384": gemms(), "xl_step_64x32x32": step(a.steps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
