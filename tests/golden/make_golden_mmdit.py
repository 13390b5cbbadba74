"""Generates tests/golden/mmdit_*.npz by EXECUTING the reference's own MMDiT source
(/root/reference/opensora/models/mmdit/{layers,math}.py, loaded by path through oracle/ref_loader.py)
on seeded inputs.  Run in the build container only (the reference does not travel to the GPU box):

    python tests/golden/make_golden_mmdit.py

The fixtures pin oracle/mmdit_oracle.py and the pieces oracle/stdit3_oracle.py shares with MMDiT."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_loader  # noqa: E402
from tests.util import save_golden, seeded_init  # noqa: E402


def ids_for(B, Lt, T, H, W):
    """img_ids / txt_ids of utils/sampling.py:437-447: (t, h, w) per image token, zeros for text."""
    img = torch.zeros(T, H, W, 3)
    img[..., 0] += torch.arange(T)[:, None, None]
    img[..., 1] += torch.arange(H)[None, :, None]
    img[..., 2] += torch.arange(W)[None, None, :]
    img = img.reshape(1, T * H * W, 3).repeat(B, 1, 1)
    return torch.cat([torch.zeros(B, Lt, 3), img], dim=1)


def main():
    layers, math_m, _ = ref_loader.load_mmdit()
    torch.manual_seed(20260922)
    C, Hh, B, Lt, T, H, W = 64, 2, 2, 5, 3, 2, 3
    D = C // Hh
    axes = [8, 12, 12]
    Li = T * H * W
    out = {}
    img, txt, vec = torch.randn(B, Li, C), torch.randn(B, Lt, C), torch.randn(B, C)
    ids = ids_for(B, Lt, T, H, W)
    pe_flux = layers.EmbedND(D, 10000, axes)(ids)
    pe_liger = layers.LigerEmbedND(D, 10000, axes)(ids)
    out.update(img=img, txt=txt, vec=vec, ids=ids, pe_flux=pe_flux, pe_liger_cos=pe_liger[0], pe_liger_sin=pe_liger[1])

    with torch.no_grad():
        # --- small pieces -------------------------------------------------------------------------
        x = torch.randn(B, Hh, Li, D)
        rn = layers.RMSNorm(D)
        seeded_init(rn, "rms")
        out.update(rms_x=x, rms_scale=rn.scale.detach(), rms_y=rn(x))
        out.update(rms_y_bf16=rn(x.bfloat16()).float())
        q, k = torch.randn(B, Hh, Lt + Li, D), torch.randn(B, Hh, Lt + Li, D)
        rq, rk = math_m.apply_rope(q, k, pe_flux)
        out.update(rope_q=q, rope_k=k, rope_q_out=rq, rope_k_out=rk)
        out.update(temb_t=torch.tensor([0.25, 0.9]), temb=layers.timestep_embedding(torch.tensor([0.25, 0.9]), 256))
        v = torch.randn(B, Hh, Lt + Li, D)
        out.update(attn_v=v, attn_out_flux=math_m.attention(q, k, v, pe_flux))

        # --- blocks -------------------------------------------------------------------------------
        for fused in (True, False):
            tag = "fused" if fused else "split"
            blk = layers.DoubleStreamBlock(C, Hh, 4.0, qkv_bias=True, fused_qkv=fused)
            seeded_init(blk, f"double_{tag}")
            oi, ot = blk(img, txt, vec, pe_flux)
            out.update({f"double_{tag}.{n}": p.detach() for n, p in blk.state_dict().items()})
            out.update({f"double_{tag}_out_img": oi, f"double_{tag}_out_txt": ot})
            sb = layers.SingleStreamBlock(C, Hh, 4.0, fused_qkv=fused)
            seeded_init(sb, f"single_{tag}")
            xcat = torch.cat((txt, img), 1)
            out.update({f"single_{tag}.{n}": p.detach() for n, p in sb.state_dict().items()})
            out.update({f"single_{tag}_out": sb(xcat, vec, pe_flux)})
        ll = layers.LastLayer(C, 1, 16)
        seeded_init(ll, "last")
        out.update({f"last.{n}": p.detach() for n, p in ll.state_dict().items()})
        out.update(last_out=ll(img, vec))
        # --- tiny full model (prepare_block_inputs + blocks + final layer), executed by the reference ---------
        _, _, model_m = layers, math_m, ref_loader.load_mmdit()[2]
        cfg = dict(in_channels=8, vec_in_dim=12, context_in_dim=20, hidden_size=C, mlp_ratio=4.0, num_heads=Hh, depth=1,
                   depth_single_blocks=1, axes_dim=axes, theta=10000, qkv_bias=True, guidance_embed=True, cond_embed=True,
                   fused_qkv=True)
        fm = model_m.Flux(device_map="cpu", torch_dtype=torch.float32, **cfg)
        seeded_init(fm, "model")
        m_img, m_cond = torch.randn(B, Li, 8), torch.randn(B, Li, 12)
        m_txt, m_y = torch.randn(B, Lt, 20), torch.randn(B, 12)
        m_t, m_g = torch.tensor([0.3, 0.8]), torch.tensor([4.0, 7.5])
        img_ids, txt_ids = ids[:, Lt:], ids[:, :Lt]
        m_out = fm(img=m_img, img_ids=img_ids, txt=m_txt, txt_ids=txt_ids, timesteps=m_t, y_vec=m_y, cond=m_cond, guidance=m_g)
        out.update({f"model.{n}": p.detach() for n, p in fm.state_dict().items()})
        out.update(model_img=m_img, model_cond=m_cond, model_txt=m_txt, model_y=m_y, model_t=m_t, model_g=m_g, model_out=m_out)
    path = os.path.join(HERE, "mmdit_blocks.npz")
    save_golden(path, out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(out), "arrays")


if __name__ == "__main__":
    main()
