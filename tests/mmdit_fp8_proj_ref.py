"""FP8-emulation reference of the MMDiT FP8 projection path (`enable_fp8(projections=True)`), for the tests.

The pinned oracle (`oracle/mmdit_oracle.py`), typically run in bf16, with the FP8 MLPs of tests/mmdit_fp8_ref.py and
every q|k|v and attention-output projection replaced by fp32 arithmetic on dequantized operands, rounded where the
product rounds:
- the q|k|v GEMM input (the LN+modulate value) per row, the weights per output channel, the bf16 q|k|v output;
- the `proj` input (the attention output) per 1 x 128 block, the weights per output channel;
- in the single blocks the same per-row LN+modulate codes feed the qkv and the mlp parts of linear1.
With tests/mmdit_fp8_attn_ref.py's `fp8_attention()` on top, the attention runs at its FP8 rounding points too.
`fp8_projections()` patches the oracle for the duration of a `with`."""
import contextlib

import torch
import torch.nn.functional as F

from tests import fp8_ref as R
from tests import mmdit_fp8_ref as MR


def _lin_rows(x, w, b):
    """The FP8 GEMM with per-row A: x quantized per row, w per output channel, bf16 output."""
    return MR._lin(R.qdq(x.float()), w, b).to(x.dtype)


def _proj(a, w, b):
    """The block-scaled FP8 GEMM of the attention output: a per 1 x 128 block, w per output channel."""
    return MR._lin(MR.qdq_blocks(a.float()), w, b).to(a.dtype)


def _qkv(M, x, W, pfx, H, fused):
    if fused:
        q, k, v = _lin_rows(x, W[pfx + "qkv.weight"], W.get(pfx + "qkv.bias")).chunk(3, dim=-1)
    else:
        q = _lin_rows(x, W[pfx + "q_proj.weight"], W.get(pfx + "q_proj.bias"))
        k = _lin_rows(x, W[pfx + "k_proj.weight"], W.get(pfx + "k_proj.bias"))
        v = _lin_rows(x, W[pfx + "v_proj.weight"], W.get(pfx + "v_proj.bias"))
    q, k, v = M._heads(q, H), M._heads(k, H), M._heads(v, H)
    q = M.rms_norm(q, W[pfx + "norm.query_norm.scale"]).to(v)
    k = M.rms_norm(k, W[pfx + "norm.key_norm.scale"]).to(v)
    return q, k, v


def _double_stream_block(M):
    def block(W, img, txt, vec, pe, num_heads, fused_qkv):
        im1s, im1c, im1g, im2s, im2c, im2g = M.modulation(vec, W["img_mod.lin.weight"], W["img_mod.lin.bias"], 6)
        tm1s, tm1c, tm1g, tm2s, tm2c, tm2g = M.modulation(vec, W["txt_mod.lin.weight"], W["txt_mod.lin.bias"], 6)
        iq, ik, iv = _qkv(M, M.ln_modulate(img, im1s, im1c), W, "img_attn.", num_heads, fused_qkv)
        tq, tk, tv = _qkv(M, M.ln_modulate(txt, tm1s, tm1c), W, "txt_attn.", num_heads, fused_qkv)
        a = M.attention(torch.cat((tq, iq), 2), torch.cat((tk, ik), 2), torch.cat((tv, iv), 2), pe)
        ta, ia = a[:, : txt.shape[1]], a[:, txt.shape[1]:]
        img = img + im1g * _proj(ia, W["img_attn.proj.weight"], W["img_attn.proj.bias"])
        img = img + im2g * M._mlp(M.ln_modulate(img, im2s, im2c), W, "img_mlp.")
        txt = txt + tm1g * _proj(ta, W["txt_attn.proj.weight"], W["txt_attn.proj.bias"])
        txt = txt + tm2g * M._mlp(M.ln_modulate(txt, tm2s, tm2c), W, "txt_mlp.")
        return img, txt
    return block


def _single_stream_block(M):
    def block(W, x, vec, pe, num_heads, fused_qkv):
        C = x.shape[-1]
        s, c, g = M.modulation(vec, W["modulation.lin.weight"], W["modulation.lin.bias"], 3)
        xm = M.ln_modulate(x, s, c)
        if fused_qkv:
            w1, b1 = W["linear1.weight"], W["linear1.bias"]
            wq, bq, wm, bm = w1[:3 * C], b1[:3 * C], w1[3 * C:], b1[3 * C:]
        else:
            wq = torch.cat((W["q_proj.weight"], W["k_proj.weight"], W["v_mlp.weight"][:C]), 0)
            bq = torch.cat((W["q_proj.bias"], W["k_proj.bias"], W["v_mlp.bias"][:C]), 0)
            wm, bm = W["v_mlp.weight"][C:], W["v_mlp.bias"][C:]
        q, k, v = _lin_rows(xm, wq, bq).chunk(3, dim=-1)
        q, k, v = M._heads(q, num_heads), M._heads(k, num_heads), M._heads(v, num_heads)
        q = M.rms_norm(q, W["norm.query_norm.scale"]).to(v)
        k = M.rms_norm(k, W["norm.key_norm.scale"]).to(v)
        a = M.attention(q, k, v, pe)
        h = F.gelu(MR._lin(R.qdq(xm.float()), wm, bm), approximate="tanh")
        out = MR._lin(MR.qdq_blocks(torch.cat((a.float(), h), -1)), W["linear2.weight"], W["linear2.bias"]).to(x.dtype)
        return x + g * out
    return block


@contextlib.contextmanager
def fp8_projections():
    """Patch oracle/mmdit_oracle.py so that `model_forward` runs every block Linear at the FP8 rounding points."""
    from oracle import mmdit_oracle as M

    saved = M._mlp, M.double_stream_block, M.single_stream_block
    M._mlp, M.double_stream_block, M.single_stream_block = MR._mlp, _double_stream_block(M), _single_stream_block(M)
    try:
        yield M
    finally:
        M._mlp, M.double_stream_block, M.single_stream_block = saved
