"""The MMDiT model at bench.py's 256px shape (B = 3, 19 + 38 blocks, C = 3072), with synthetic weights, for the FP8
measurements (tests/mmdit_fp8_bench.py)."""
import torch


def mmdit_256px():
    from bench import MMDIT_256PX
    from opensora.models.mmdit.model import MMDiTConfig, MMDiTModel

    cfg = MMDIT_256PX
    B, T, H, W, Lt = 3, 33, 12, 21, 512
    Li = T * H * W
    torch.manual_seed(0)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            net = MMDiTModel(MMDiTConfig(from_pretrained=None, cache_dir=None, **cfg)).eval()
    finally:
        torch.set_default_dtype(prev)
    with torch.no_grad():
        torch.nn.init.normal_(net.cond_in.weight, std=0.02)
    g = torch.Generator(device="cuda").manual_seed(5)
    rb = lambda *s: torch.randn(*s, device="cuda", generator=g).to(torch.bfloat16)   # noqa: E731
    ids = torch.stack(torch.meshgrid(torch.arange(T), torch.arange(H), torch.arange(W), indexing="ij"), -1).reshape(1, Li, 3)
    inp = dict(img=rb(B, Li, 64), img_ids=ids.float().repeat(B, 1, 1).cuda().to(torch.bfloat16), txt=rb(B, Lt, 4096),
               txt_ids=torch.zeros(B, Lt, 3, device="cuda", dtype=torch.bfloat16),
               timesteps=torch.full((B,), 0.7, device="cuda", dtype=torch.bfloat16), y_vec=rb(B, 768), cond=rb(B, Li, 68),
               guidance=None)
    return net, inp
