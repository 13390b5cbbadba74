"""Measurement of the FP8 projections of MMDiT on one GPU; prints one JSON line.

  python tests/mmdit_fp8_proj_bench.py [--reps 6] [--iters 5] [--no-model]

1. Per op at M = 26 484 rows (B = 3 x L = 8 828, C = 3072), bf16 against FP8, alternated windows, medians and spreads:
   the q|k|v GEMM (3072 -> 9216, bias) on bf16 A against per-row e4m3 A; the attention-output projection (3072 -> 3072,
   bias + gate + residual) on bf16 A against block-scaled e4m3 A; the FP8 attention (B 3, L 8 828, H 24) with bf16 output
   (osb_attn_fp8) against e4m3 + block-scale output (osb_attn_fp8_blocks).
2. The whole 256px forward (bench.py's mmdit leg, 19 + 38 blocks) in three modes on one model object, alternated,
   median: bf16; FP8 MLPs + FP8 attention; the same plus FP8 projections.  The rel-L2 of each FP8 output against bf16.
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

from tests.models import B_256PX as B, L_256PX as L, LT_256PX as LT, mmdit_256px  # noqa: E402
from tests.timing import alternate, card, window_ms  # noqa: E402

C, H = 3072, 24


def ops(reps, iters):
    import osb200

    g = torch.Generator(device="cuda").manual_seed(0)
    M = B * L
    rb = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).to(torch.bfloat16)   # noqa: E731
    x = rb(M, C)
    res = {}
    # q|k|v: LN+modulate output (bf16 / e4m3 + row scales) -> [M, 3C]
    wq, bq = rb(3 * C, C, sc=0.02), rb(3 * C, sc=0.02)
    x8, xs = osb200.quant_rows_fp8(x)
    wq8, sq = osb200.quant_blocks_fp8(wq, block=C)
    sq = sq.view(-1)
    out = torch.empty(M, 3 * C, dtype=torch.bfloat16, device="cuda")
    t = alternate({"bf16": lambda: osb200.gemm(x, wq, bq, out=out),
                    "fp8": lambda: osb200.gemm_fp8_blocks(x8, xs, wq8, sq, bq, out=out)}, reps, iters)
    t.update(TF_per_s_bf16=round(2.0 * M * 3 * C * C / t["bf16"] / 1e9, 1),
             TF_per_s_fp8=round(2.0 * M * 3 * C * C / t["fp8"] / 1e9, 1), speedup=round(t["bf16"] / t["fp8"], 3))
    res["qkv_gemm_M26484_3072x9216"] = t
    # proj: attention output -> x + gate * (W a + b)
    wp, bp, res_x = rb(C, C, sc=0.02), rb(C, sc=0.02), rb(M, C)
    gate = torch.randn(1, C, device="cuda", generator=g)
    a8, as_ = osb200.quant_blocks_fp8(x)
    wp8, sp = osb200.quant_blocks_fp8(wp, block=C)
    sp = sp.view(-1)
    out = torch.empty(M, C, dtype=torch.bfloat16, device="cuda")
    kw = dict(epilogue=osb200.EPI_BIAS_GATE_RES, residual=res_x, gate=gate, out=out)
    t = alternate({"bf16": lambda: osb200.gemm(x, wp, bp, **kw),
                    "fp8": lambda: osb200.gemm_fp8_blocks(a8, as_, wp8, sp, bp, **kw)}, reps, iters)
    t.update(TF_per_s_bf16=round(2.0 * M * C * C / t["bf16"] / 1e9, 1),
             TF_per_s_fp8=round(2.0 * M * C * C / t["fp8"] / 1e9, 1), speedup=round(t["bf16"] / t["fp8"], 3))
    res["proj_gemm_gate_res_M26484_3072x3072"] = t
    # the FP8 attention, bf16 output against e4m3 + block scales into the [rows, 5C] cat buffer
    D = 128
    qkv = rb(M, 3 * C)
    w = [(1 + 0.2 * torch.randn(D, device="cuda", generator=g)).to(torch.bfloat16) for _ in range(4)]
    ang = torch.rand(L, D // 2, device="cuda", generator=g) * 6.28
    akw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
               head_dim=D, q_norm_w=w[0], k_norm_w=w[1], q_norm_w2=w[2], k_norm_w2=w[3], norm_split=LT,
               rope_cos=torch.cos(ang), rope_sin=torch.sin(ang), rope_half=True)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    ws = osb200.attn_fp8_workspace(B, L, H, "cuda")
    out_bf = torch.empty(M, C, dtype=torch.bfloat16, device="cuda")
    cat8 = torch.empty(M, 5 * C, dtype=torch.float8_e4m3fn, device="cuda")
    cats = torch.empty(M, 5 * C // 128, device="cuda")
    t = alternate({"bf16_out": lambda: osb200.attn_fp8(q, k, v, out_bf, workspace=ws, **akw),
                    "fp8_out": lambda: osb200.attn_fp8_blocks(q, k, v, cat8[:, :C], cats[:, :H], workspace=ws, **akw),
                    "bf16_out_then_quant_blocks": lambda: (osb200.attn_fp8(q, k, v, out_bf, workspace=ws, **akw),
                                                           osb200.quant_blocks_fp8(out_bf, out=cat8[:, :C],
                                                                                   out_scale=cats[:, :H]))},
                   reps, iters)
    deq = (cat8[:, :C].float().view(M, H, D) * cats[:, :H, None]).view(M, C)
    t["fp8_out_dequantized_vs_bf16_out_rel_l2"] = float((deq - out_bf.float()).norm() / out_bf.float().norm())
    res["attn_fp8_B3_L8828_H24"] = t
    return res


def model(net, inp, reps):
    modes = {"bf16": (False, False), "fp8_mlps_attention": (True, False), "fp8_mlps_attention_projections": (True, True)}

    def setmode(m):
        on, proj = modes[m]
        (net.enable_fp8_attention if on else net.disable_fp8_attention)()
        if on:
            net.enable_fp8(projections=proj)
        else:
            net.disable_fp8()

    res, outs = {}, {}
    t = {m: [] for m in modes}
    with torch.no_grad():
        for m in modes:
            setmode(m)
            outs[m] = net(**inp).float()
        for m in ("fp8_mlps_attention", "fp8_mlps_attention_projections"):
            res[f"{m}_vs_bf16_rel_l2"] = float((outs[m] - outs["bf16"]).norm() / outs["bf16"].norm())
        for i in range(reps):
            for m in (list(modes) if i % 2 == 0 else list(modes)[::-1]):
                setmode(m)
                net(**inp)   # quantizes the weights / warms the workspaces off the clock
                t[m].append(window_ms(lambda: net(**inp), 1))
        setmode("bf16")
    res.update({f"{m}_ms": round(statistics.median(v), 2) for m, v in t.items()})
    res.update({f"{m}_spread_ms": round(max(v) - min(v), 2) for m, v in t.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mmdit_fp8_proj_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
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
