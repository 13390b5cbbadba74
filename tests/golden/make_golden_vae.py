"""Generates tests/golden/vae_blocks.npz by EXECUTING the reference's own causal-VAE source
(/root/reference/opensora/models/hunyuan_vae/{unet_causal_3d_blocks,vae}.py + models/vae/utils.py, loaded by
path through oracle/ref_loader.py; diffusers stand-ins documented there).  Build container only:

    python tests/golden/make_golden_vae.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_loader  # noqa: E402
from tests.util import save_golden, seeded_init  # noqa: E402


def main():
    blocks, vae = ref_loader.load_hunyuan_vae()
    g = torch.Generator().manual_seed(20260922)
    torch.manual_seed(20260922)
    out = {}
    with torch.no_grad():
        x = torch.randn(1, 8, 5, 6, 10, generator=g)
        out["conv_x"] = x
        for tag, stride in (("s111", (1, 1, 1)), ("s122", (1, 2, 2)), ("s222", (2, 2, 2))):
            c = blocks.CausalConv3d(8, 16, 3, stride=stride)
            seeded_init(c, f"conv_{tag}")
            out.update({f"conv_{tag}.w": c.conv.weight, f"conv_{tag}.b": c.conv.bias, f"conv_{tag}.y": c(x)})
        c1 = blocks.CausalConv3d(8, 16, 1)
        seeded_init(c1, "conv_k1")
        out.update({"conv_k1.w": c1.conv.weight, "conv_k1.b": c1.conv.bias, "conv_k1.y": c1(x)})
        for tag, f in (("u222", (2, 2, 2)), ("u122", (1, 2, 2))):
            up = blocks.UpsampleCausal3D(8, out_channels=8, upsample_factor=f)
            seeded_init(up, f"up_{tag}")
            out.update({f"up_{tag}.w": up.conv.conv.weight, f"up_{tag}.b": up.conv.conv.bias, f"up_{tag}.y": up(x)})
        xr = torch.randn(1, 16, 3, 6, 6, generator=g)
        out["res_x"] = xr
        for tag, co in (("same", 16), ("wide", 32)):
            r = blocks.ResnetBlockCausal3D(in_channels=16, out_channels=co, groups=4)
            seeded_init(r, f"res_{tag}")
            out.update({f"res_{tag}.{n}": p for n, p in r.state_dict().items()})
            out[f"res_{tag}.y"] = r(xr)
        mb = blocks.UNetMidBlockCausal3D(in_channels=16, attention_head_dim=16, resnet_groups=4)
        seeded_init(mb, "mid")
        mask = blocks.prepare_causal_attention_mask(3, 36, xr.dtype, xr.device, batch_size=1)
        out.update({f"mid.{n}": p for n, p in mb.state_dict().items()})
        out["mid.y"] = mb(xr, mask)
        chans = (16, 32, 32, 32)
        enc = vae.EncoderCausal3D(in_channels=3, out_channels=4, block_out_channels=chans, layers_per_block=1, norm_num_groups=4)
        dec = vae.DecoderCausal3D(in_channels=4, out_channels=3, block_out_channels=chans, layers_per_block=1, norm_num_groups=4)
        seeded_init(enc, "enc")
        seeded_init(dec, "dec")
        v = torch.randn(1, 3, 9, 32, 32, generator=g)
        z = enc(v)
        y = dec(z[:, :4])
        out.update({f"enc.{n}": p for n, p in enc.state_dict().items()})
        out.update({f"dec.{n}": p for n, p in dec.state_dict().items()})
        out.update(enc_x=v, enc_y=z, dec_y=y)
    path = os.path.join(HERE, "vae_blocks.npz")
    save_golden(path, out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(out), "arrays")


if __name__ == "__main__":
    main()
