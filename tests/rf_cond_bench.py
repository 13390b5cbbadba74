"""Measurement of image / video conditioning on one GPU; prints one JSON line.

  python tests/rf_cond_bench.py [--steps 5] [--reps 5]

- osb_rf_masked_step kernel time (CUDA-graph replay of 200 launches) and achieved bandwidth at [1,4,64,32,32] and
  [2,4,128,90,160], next to osb_cfg_euler on the same latent.  The step is the image-to-video one (frame 0 kept, in
  place): algorithmic bytes = 8 per element of the updated frames (read cond, uncond, z; write z); the t2v step moves 8
  per element of every frame.
- STDiT3-XL/2 at 64x32x32 (CFG forward batch 2): ms per sampling step of the conditioned loop (strategy "0") and of the
  text-to-video loop, alternated, after a warm-up, median and spread over --reps runs of --steps steps.
- The same model's forward (batch 2) with and without x_mask, alternated.
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

from tests.timing import card, window_ms  # noqa: E402


def kernel(shape, iters=200):
    import osb200

    g = torch.Generator(device="cuda").manual_seed(0)
    B, C, T, H, W = shape
    vc, vu, z, noise = (torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4))
    fm = torch.ones(B, T, device="cuda")
    fm[:, 0] = 0
    tc, tn = torch.full((B,), 750.0, device="cuda"), torch.full((B,), 500.0, device="cuda")
    launches = {
        "masked": lambda: osb200.rf_masked_step(vc, vu, z, fm, tc, tn, guidance=7.0, noise=noise, out=z),
        "t2v": lambda: osb200.cfg_euler(vc, vu, None, z, g_txt=7.0, dt=-0.0, out=z),     # dt 0: z stays finite
    }
    # `iters` launches captured in one CUDA graph: the replay times the kernels, not the Python binding around them
    graphs = {}
    for k, f in launches.items():
        f()
        graphs[k] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[k]):
            for _ in range(iters):
                f()
        graphs[k].replay()
    ms_m, ms_c = [], []
    for _ in range(5):
        ms_m.append(window_ms(graphs["masked"].replay, 1) / iters)
        ms_c.append(window_ms(graphs["t2v"].replay, 1) / iters)
    n = z.numel()
    bytes_m, bytes_c = 8.0 * n * (T - 1) / T, 8.0 * n
    m, c = statistics.median(ms_m), statistics.median(ms_c)
    return {"shape": list(shape), "rf_masked_step_us": round(m * 1e3, 2), "rf_masked_step_GBps": round(bytes_m / m / 1e6, 1),
            "rf_masked_step_us_spread": [round(min(ms_m) * 1e3, 2), round(max(ms_m) * 1e3, 2)],
            "cfg_euler_us": round(c * 1e3, 2), "cfg_euler_GBps": round(bytes_c / c / 1e6, 1)}


def model_legs(steps, reps):
    from opensora.schedulers import RFLOW
    from opensora.utils.inference_utils import apply_mask_strategy
    from tests.models import stdit3_inputs, stdit3_pair

    prod, _, cfg = stdit3_pair("xl")
    B = 1
    inp = stdit3_inputs(cfg, B, 64, 32, 32, lens=[260], device="cuda")
    z = inp["x"].to(torch.bfloat16)
    ref = [[torch.randn(cfg.in_channels, 1, 32, 32, device="cuda")]]
    zc = z.clone()
    fm = apply_mask_strategy(zc, ref, ["0"], loop_i=0)
    y_null = prod.y_embedder.y_embedding.detach()[None, None].repeat(B, 1, 1, 1)
    extra = dict(fps=inp["fps"], height=inp["height"], width=inp["width"])
    sch = RFLOW(num_sampling_steps=steps, cfg_scale=7.0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    run = {
        "t2v": lambda: sch.sample(prod, z, inp["y"], y_null, mask=inp["mask"], additional_args=extra),
        "i2v": lambda: sch.sample(prod, zc, inp["y"], y_null, mask=inp["mask"], additional_args=extra, frame_mask=fm,
                                  generator=gen),
    }
    x2 = torch.cat((z, z))
    t2 = torch.full((2,), 750.0, device="cuda")
    kw2 = dict(y=torch.cat((inp["y"], y_null)), mask=torch.cat((inp["mask"], inp["mask"])), fps=inp["fps"].repeat(2),
               height=inp["height"].repeat(2), width=inp["width"].repeat(2))
    xm = fm.ge(0.75).repeat(2, 1)
    fwd = {"forward": lambda: prod(x2, t2, **kw2), "forward_x_mask": lambda: prod(x2, t2, x_mask=xm, **kw2)}
    res = {}
    with torch.no_grad():
        for legs, n, per in ((run, 1, steps), (fwd, 3, 1)):
            for f in legs.values():      # warm-up
                f()
            times = {k: [] for k in legs}
            for _ in range(reps):
                for k, f in legs.items():
                    times[k].append(window_ms(f, n) / per)
            for k, v in times.items():
                res[k + "_ms"] = round(statistics.median(v), 2)
                res[k + "_ms_spread"] = [round(min(v), 2), round(max(v), 2)]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rf_cond_bench needs a CUDA device")
    name, power = card()
    out = {"gpu": name, "power_limit_and_max_sm_clock": power,
           "kernel": [kernel((1, 4, 64, 32, 32)), kernel((2, 4, 128, 90, 160))],
           "stdit3_xl_64x32x32": dict(model_legs(a.steps, a.reps), steps_per_run=a.steps, cfg_batch=2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
