"""VAE leg of BASELINE.json's metric: encode / decode fps of the causal 3D VAE on a synthetic video (bench.py runs
33x720x1280: untiled, bf16, one H100).  Usable at any size: python tests/vae_bench.py T H W [iters]."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "open-sora_b200"))
import torch

ENC_TF, DEC_TF = 545.8, 1017.9  # algorithmic conv TFLOP at 65x720x1280 (SURVEY.md §8d)


def run(T=65, H=720, W=1280, iters=2, do_encode=True):
    import osb200
    from opensora.registry import MODELS, build_module

    torch.manual_seed(0)
    with torch.device("cuda"):  # initialise the 246 M parameters on the device, not on the host
        vae = build_module(dict(type="hunyuan_vae"), MODELS, device_map="cuda").eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    lt, lh, lw = vae.get_latent_size([T, H, W])
    z = torch.randn(1, 16, lt, lh, lw, device="cuda", generator=g).to(torch.bfloat16)
    res = {"video": [T, H, W], "latent": [lt, lh, lw]}
    with torch.no_grad():
        out = vae.decode(z)  # warm-up (packs weights)
        torch.cuda.synchronize()
        l0 = osb200.launch_count()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            out = vae.decode(z)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / iters
        scale = (T * H * W) / (65 * 720 * 1280)
        res.update(decode_ms=ms, decode_fps=T / (ms / 1e3), decode_conv_tflops=DEC_TF * scale / (ms / 1e3),
                   decode_launches=(osb200.launch_count() - l0) // iters, out_shape=list(out.shape),
                   finite=bool(torch.isfinite(out).all()), peak_gb=torch.cuda.max_memory_allocated() / 2**30)
        if do_encode:
            del out
            x = (torch.rand(1, 3, T, H, W, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
            zz = vae.encode(x, sample_posterior=False)
            torch.cuda.synchronize()
            s.record()
            for _ in range(iters):
                zz = vae.encode(x, sample_posterior=False)
            e.record()
            torch.cuda.synchronize()
            ms = s.elapsed_time(e) / iters
            res.update(encode_ms=ms, encode_fps=T / (ms / 1e3), encode_conv_tflops=ENC_TF * scale / (ms / 1e3),
                       peak_gb=torch.cuda.max_memory_allocated() / 2**30)
    return res


if __name__ == "__main__":
    a = [int(v) for v in sys.argv[1:]]
    T, H, W = (a + [65, 720, 1280])[:3] if len(a) >= 3 else (65, 720, 1280)
    it = a[3] if len(a) > 3 else 2
    if "--profile" in os.environ.get("VAE_BENCH_FLAGS", ""):
        import osb200

        osb200.start_profile()
    print(json.dumps(run(T, H, W, it)))
