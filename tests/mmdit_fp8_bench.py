"""Measurement of the block-scaled FP8 MLPs of MMDiT on one GPU; prints one JSON line.

  python tests/mmdit_fp8_bench.py [--reps 6] [--iters 10] [--no-model]

- At the 256px inference shape (M = 26 484 token rows, C = 3072), bf16 against FP8, alternated windows, median of --reps
  windows of --iters calls:
  - fc1 3072 -> 12 288: bf16 GEMM + GELU against the FP8 GEMM whose epilogue emits e4m3 codes and block scales;
  - fc2 12 288 -> 3072 (gate + residual): bf16 against the block-scaled FP8 GEMM;
  - the mlp part of linear1 (3072 -> 12 288 + GELU into the cat buffer): bf16 against ln_modulate_fp8 + the FP8 GEMM
    (the bf16 side shares the qkv part's LN+modulate, so the FP8 side pays its second LN pass here);
  - linear2 15 360 -> 3072: bf16 against the attention-output block quantizer + the block-scaled FP8 GEMM.
- The whole MMDiT 256px forward (bench.py's mmdit leg: B = 3, 19 + 38 blocks), FP8 off against on, same model object,
  alternated, median.
The card's name, power limit and max SM clock are read in the same run."""
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

from tests.models import ROWS_256PX as M_ROWS, mmdit_256px  # noqa: E402
from tests.timing import alternate, card, window_ms  # noqa: E402


def gemms(reps, iters):
    import osb200 as osb

    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).to(torch.bfloat16)   # noqa: E731
    M, C, H4 = M_ROWS, 3072, 12288
    f8 = torch.float8_e4m3fn
    x, res = rn(M, C), rn(M, C)
    shift, scale, gate = (torch.randn(1, C, device="cuda", generator=g) * 0.1 for _ in range(3))
    w1, b1, w2, b2 = rn(H4, C, sc=C ** -0.5), rn(H4, sc=0.1), rn(C, H4, sc=H4 ** -0.5), rn(C, sc=0.1)
    wl2 = rn(C, C + H4, sc=(C + H4) ** -0.5)
    q1, q2, ql2 = (osb.quant_blocks_fp8(w, block=w.shape[1]) for w in (w1, w2, wl2))
    xm = osb.ln_modulate(x, shift, scale, group_rows=M)
    x8, xs = osb.ln_modulate_fp8(x, shift, scale, group_rows=M)
    h = torch.empty(M, H4, dtype=torch.bfloat16, device="cuda")
    h8, hs = torch.empty(M, H4, dtype=f8, device="cuda"), torch.empty(M, H4 // 128, device="cuda")
    cat = rn(M, C + H4)
    cat8, cats = torch.empty(M, C + H4, dtype=f8, device="cuda"), torch.empty(M, (C + H4) // 128, device="cuda")
    out = torch.empty(M, C, dtype=torch.bfloat16, device="cuda")
    ao = cat[:, :C]
    osb.gemm_fp8_blocks(x8, xs, q1[0], q1[1].view(-1), b1, epilogue=osb.EPI_BIAS_GELU_TANH_FP8, out=h8, out_scale=hs)
    osb.quant_blocks_fp8(ao, out=cat8[:, :C], out_scale=cats[:, :C // 128])
    osb.gemm_fp8_blocks(x8, xs, q1[0], q1[1].view(-1), b1, epilogue=osb.EPI_BIAS_GELU_TANH_FP8, out=cat8[:, C:],
                        out_scale=cats[:, C // 128:])
    cases = {
        "fc1_3072x12288": {
            "bf16": lambda: osb.gemm(xm, w1, b1, epilogue=osb.EPI_BIAS_GELU_TANH, out=h),
            "fp8": lambda: osb.gemm_fp8_blocks(x8, xs, q1[0], q1[1].view(-1), b1, epilogue=osb.EPI_BIAS_GELU_TANH_FP8,
                                               out=h8, out_scale=hs)},
        "fc2_12288x3072": {
            "bf16": lambda: osb.gemm(h, w2, b2, epilogue=osb.EPI_BIAS_GATE_RES, residual=res, gate=gate, out=out),
            "fp8": lambda: osb.gemm_fp8_blocks(h8, hs, q2[0], q2[1].view(-1), b2, epilogue=osb.EPI_BIAS_GATE_RES,
                                               residual=res, gate=gate, out=out)},
        "linear1_mlp_part": {
            "bf16": lambda: osb.gemm(xm, w1, b1, epilogue=osb.EPI_BIAS_GELU_TANH, out=cat[:, C:]),
            "fp8": lambda: (osb.ln_modulate_fp8(x, shift, scale, group_rows=M, out=x8, out_scale=xs),
                            osb.gemm_fp8_blocks(x8, xs, q1[0], q1[1].view(-1), b1, epilogue=osb.EPI_BIAS_GELU_TANH_FP8,
                                                out=cat8[:, C:], out_scale=cats[:, C // 128:]))},
        "linear2_15360x3072_with_quantizer": {
            "bf16": lambda: osb.gemm(cat, wl2, b2, epilogue=osb.EPI_BIAS_GATE_RES, residual=res, gate=gate, out=out),
            "fp8": lambda: (osb.quant_blocks_fp8(ao, out=cat8[:, :C], out_scale=cats[:, :C // 128]),
                            osb.gemm_fp8_blocks(cat8, cats, ql2[0], ql2[1].view(-1), b2, epilogue=osb.EPI_BIAS_GATE_RES,
                                                residual=res, gate=gate, out=out))},
        "attn_out_quantizer_alone": {
            "fp8": lambda: osb.quant_blocks_fp8(ao, out=cat8[:, :C], out_scale=cats[:, :C // 128])},
        "ln_modulate_fp8_alone": {
            "fp8": lambda: osb.ln_modulate_fp8(x, shift, scale, group_rows=M, out=x8, out_scale=xs)},
    }
    r = {}
    for name, fns in cases.items():
        t = alternate(fns, reps, iters)
        if "bf16" in t:
            t["fp8_over_bf16"] = round(t["fp8"] / t["bf16"], 3)
        r[name] = t
    return r


def model(reps):
    net, inp = mmdit_256px()
    res = {}
    with torch.no_grad():
        plain = net(**inp).float()
        net.enable_fp8()
        fp8 = net(**inp).float()
        res["fp8_vs_bf16_rel_l2"] = float((fp8 - plain).norm() / plain.norm())
        res["finite"] = bool(torch.isfinite(fp8).all())
        t = {"bf16": [], "fp8": []}
        for i in range(reps):
            for k in (("bf16", "fp8") if i % 2 == 0 else ("fp8", "bf16")):
                if k == "fp8":
                    net.enable_fp8()
                else:
                    net.disable_fp8()
                net(**inp)   # quantizes the weights / warms the workspaces off the clock
                t[k].append(window_ms(lambda: net(**inp), 1))
        net.disable_fp8()
    res.update({f"{k}_ms": round(statistics.median(v), 2) for k, v in t.items()})
    res.update({f"{k}_spread_ms": round(max(v) - min(v), 2) for k, v in t.items()})
    res["fp8_gain_pct"] = round(100.0 * (1.0 - res["fp8_ms"] / res["bf16_ms"]), 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mmdit_fp8_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
    import osb200

    osb200.init(0)
    name, power = card()
    res = {"card": name, "power_limit,max_sm_clock": power, "rows": M_ROWS, "gemm_ms": gemms(a.reps, a.iters)}
    if not a.no_model:
        res["mmdit_256px_forward"] = model(a.reps)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
