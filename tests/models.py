"""Seeded models and inputs shared by the tests and the measurement scripts: STDiT3 product / oracle pairs, the small
MMDiT (and its full-width variant), the MMDiT at bench.py's 256px shape, the reference-class block case and the small
causal VAE of the goldens."""
import torch

# ---- STDiT3 -------------------------------------------------------------------------------------------------------------


def stdit3_pair(name: str = "xs", device="cuda", seed=1234):
    """(product model in bf16 on `device`, fp32 oracle holding the SAME bf16-rounded weights, oracle config).

    "xs" is STDiT3-XS/2 as shipped (4 heads of 72); "xs64" is the XS/2 plumbing size at hidden size 256 (4 heads of 64),
    for the FP8 paths, which need hidden sizes that are multiples of 128; "xl" is STDiT3-XL/2."""
    from opensora.models.stdit.stdit3 import STDiT3 as Product, STDiT3Config as PCfg
    from oracle import stdit3_oracle as O

    ocfg = {"xs": O.STDiT3_XS_2_config, "xl": O.STDiT3_XL_2_config,
            "xs64": lambda: O.STDiT3Config(depth=2, hidden_size=256, patch_size=(1, 2, 2), num_heads=4)}[name]()
    oracle = O.STDiT3(ocfg).eval()
    O.init_synthetic_weights(oracle, seed)
    sd = {k: v.to(torch.bfloat16) for k, v in oracle.state_dict().items()}
    oracle.load_state_dict({k: v.float() for k, v in sd.items()})
    prod = Product(PCfg(depth=ocfg.depth, hidden_size=ocfg.hidden_size, num_heads=ocfg.num_heads,
                        patch_size=ocfg.patch_size)).eval()
    prod.load_state_dict(sd)
    return prod.to(device=device, dtype=torch.bfloat16), oracle, ocfg


def stdit3_inputs(cfg, B, T, H, W, lens=None, device="cpu"):
    """The oracle's synthetic inputs with every float rounded to bf16 (kept in fp32), on `device`."""
    from oracle import stdit3_oracle as O

    inp = O.synthetic_inputs(cfg, B=B, T=T, H=H, W=W, lens=lens)
    return {k: (v.to(torch.bfloat16).float() if v.is_floating_point() else v).to(device) for k, v in inp.items()}


# ---- MMDiT ---------------------------------------------------------------------------------------------------------------
MMDIT_CFG = dict(in_channels=64, vec_in_dim=96, context_in_dim=128, hidden_size=256, mlp_ratio=4.0, num_heads=2, depth=2,
                 depth_single_blocks=2, axes_dim=[16, 56, 56], theta=10000, qkv_bias=True, guidance_embed=True,
                 cond_embed=True)
# the full-width variant: C = 3072 in 24 heads of 128, still 2 double + 2 single blocks
MMDIT_WIDE = dict(hidden_size=3072, num_heads=24)


def mmdit_ids(B, Lt, T, H, W):
    img = torch.zeros(T, H, W, 3)
    img[..., 0] += torch.arange(T)[:, None, None]
    img[..., 1] += torch.arange(H)[None, :, None]
    img[..., 2] += torch.arange(W)[None, None, :]
    return torch.zeros(B, Lt, 3), img.reshape(1, T * H * W, 3).repeat(B, 1, 1)


def mmdit_model(fused=True, liger=False, device="cpu", **cfg_overrides):
    """MMDIT_CFG (with `cfg_overrides`) built through the registry with seeded weights, in bf16 on `device`: norm scales
    1 + 0.2 N(0, 1), vectors and the conditioning input 0.05 N(0, 1), other matrices as the model initialises them."""
    from opensora.registry import MODELS, build_module

    torch.manual_seed(7)
    m = build_module(dict(type="flux", **dict(MMDIT_CFG, **cfg_overrides), fused_qkv=fused, use_liger_rope=liger),
                     MODELS, device_map="cpu", torch_dtype=torch.float32)
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("scale"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 or "cond_in" in n:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
    return m.to(device).to(torch.bfloat16)


def mmdit_inputs(B=2, Lt=24, thw=(2, 4, 6), ctx=128, seed=3, guidance=4.0):
    """Seeded bf16 MMDiT inputs on the CPU; timesteps spread over [0.3, 0.8].  `guidance` is one value for every sample
    or a list of per-sample values."""
    T, H, W = thw
    g = torch.Generator().manual_seed(seed)
    rb = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)  # noqa: E731
    txt_ids, img_ids = mmdit_ids(B, Lt, T, H, W)
    return dict(img=rb(B, T * H * W, 64), img_ids=img_ids, txt=rb(B, Lt, ctx), txt_ids=txt_ids,
                timesteps=torch.linspace(0.3, 0.8, B), y_vec=rb(B, 96), cond=rb(B, T * H * W, 68),
                guidance=torch.full((B,), guidance) if isinstance(guidance, float) else torch.tensor(guidance))


# bench.py's 256px MMDiT forward: B = 3 samples of L = 512 text + 33 x 12 x 21 latent tokens, C = 3072 in 24 heads of 128
B_256PX, LT_256PX, THW_256PX = 3, 512, (33, 12, 21)
L_256PX = LT_256PX + THW_256PX[0] * THW_256PX[1] * THW_256PX[2]
ROWS_256PX = B_256PX * L_256PX
# (K, N) of the block Linears at C = 3072
GEMMS_256PX = {"qkv": (3072, 9216), "proj": (3072, 3072), "mlp_up": (3072, 12288), "mlp_down": (12288, 3072),
               "linear1": (3072, 21504), "linear2": (15360, 3072)}


def mmdit_256px():
    """The MMDiT model at bench.py's 256px shape (19 + 38 blocks) with synthetic bf16 weights on the GPU, and its inputs."""
    from bench import MMDIT_256PX
    from opensora.models.mmdit.model import MMDiTConfig, MMDiTModel

    B, Lt, (T, H, W) = B_256PX, LT_256PX, THW_256PX
    Li = T * H * W
    torch.manual_seed(0)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            net = MMDiTModel(MMDiTConfig(from_pretrained=None, cache_dir=None, **MMDIT_256PX)).eval()
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


TOKEN_STRIDE = 3   # tests/golden/ref_classes.npz keeps every third token of the reference outputs (float16)


def mmdit_block_case(L, fused):
    """Seeded DoubleStreamBlock / SingleStreamBlock (C = 256, 2 heads) built from the layers module `L` (the reference's
    mmdit/layers.py executed by path, or the in-tree mirror, which draws identical parameters) and their inputs."""
    torch.manual_seed(5)
    C, H, B, Lt, Li = 256, 2, 2, 24, 48
    dbl = L.DoubleStreamBlock(C, H, mlp_ratio=4.0, qkv_bias=True, fused_qkv=fused).eval()
    sgl = L.SingleStreamBlock(C, H, mlp_ratio=4.0, fused_qkv=fused).eval()
    with torch.no_grad():
        for blk in (dbl, sgl):
            for n, p in blk.named_parameters():
                p.copy_(torch.randn_like(p) * (0.2 if n.endswith("scale") else 0.05) + (1.0 if n.endswith("scale") else 0.0))
    ids = torch.zeros(B, Lt + Li, 3)
    ids[:, Lt:, 0] = torch.arange(Li) // 16
    ids[:, Lt:, 1] = (torch.arange(Li) // 4) % 4
    ids[:, Lt:, 2] = torch.arange(Li) % 4
    pe = L.EmbedND(dim=C // H, theta=10000, axes_dim=[16, 56, 56])(ids)
    bf = torch.bfloat16
    img, txt, vec = torch.randn(B, Li, C).to(bf), torch.randn(B, Lt, C).to(bf), torch.randn(B, C).to(bf)
    return dbl, sgl, pe, img, txt, vec


# ---- causal VAE ----------------------------------------------------------------------------------------------------------


def tiny_vae(G, **kw):
    """The small hunyuan_vae of tests/golden/vae_blocks.npz (fp32, CPU) with the golden's encoder / decoder weights."""
    from opensora.registry import MODELS, build_module

    m = build_module(dict(type="hunyuan_vae", block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=4,
                          latent_channels=4, **kw), MODELS, device_map="cpu")
    m.encoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("enc.")})
    m.decoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("dec.")})
    return m


def posterior_inputs():
    """Seeded (parameters, second parameters) pairs: 5-D latent, 4-D image and token-shaped distributions."""
    g = torch.Generator().manual_seed(5)
    out = []
    for shape in ((2, 8, 3, 4, 5), (2, 8, 6, 7), (2, 9, 8)):
        par = torch.randn(*shape, generator=g) * 3.0
        par2 = torch.randn(*shape, generator=g)
        out.append((par, par2))
    return out
