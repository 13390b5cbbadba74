"""Generates tests/golden/vae_tiled.npz by EXECUTING the reference's own `AutoencoderKLCausal3D`
(hunyuan_vae/autoencoder_kl_causal_3d.py, loaded by path with the diffusers plumbing stubbed, oracle/ref_loader.py) in
its tiled / blended modes (:384-552).  Encoder / decoder weights are the ones already stored in vae_blocks.npz.
Build container only."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_loader  # noqa: E402
from tests.util import load_golden, save_golden  # noqa: E402


def main():
    _, _, ae = ref_loader.load_hunyuan_vae(True)
    G = load_golden("vae_blocks.npz")
    cfg = ae.AutoEncoder3DConfig(from_pretrained=None, latent_channels=4, layers_per_block=1, norm_num_groups=4,
                                 block_out_channels=(16, 32, 32, 32), sample_size=32, sample_tsize=8)
    m = ae.AutoencoderKLCausal3D(cfg).eval()
    m.encoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("enc.")})
    m.decoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("dec.")})
    g = torch.Generator().manual_seed(77)
    out = {}
    with torch.no_grad():
        for n, p in list(m.quant_conv.named_parameters()) + list(m.post_quant_conv.named_parameters()):
            p.copy_(torch.randn(p.shape, generator=g) * 0.3)
        out.update(quant_w=m.quant_conv.weight, quant_b=m.quant_conv.bias, post_w=m.post_quant_conv.weight,
                   post_b=m.post_quant_conv.bias)
        x = torch.randn(1, 3, 13, 48, 40, generator=g).half().float()   # stored as float16: exact
        out["x"] = x
        for tag, sp, tp in (("none", False, False), ("spatial", True, False), ("temporal", False, True), ("both", True, True)):
            m.enable_spatial_tiling(sp)
            m.enable_temporal_tiling(tp)
            z = m.encode(x, sample_posterior=False)
            y = m.decode(z)
            out[f"z_{tag}"] = z
            out[f"y_{tag}"] = y
    path = os.path.join(HERE, "vae_tiled.npz")
    # the decoded videos are stored in float16 (relative error 2^-11, far inside the 2e-3 of the comparisons)
    save_golden(path, out, half={"x"} | {k for k in out if k.startswith("y_")})
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", {k: tuple(v.shape) for k, v in out.items() if k[0] in "zy"})


if __name__ == "__main__":
    main()
