"""FP8-emulation reference of the MMDiT FP8 MLP path (include/osb200.h, osb_gemm_fp8_blocks), for the tests.

The pinned oracle (`oracle/mmdit_oracle.py`), typically run in bf16, with every block MLP replaced by fp32 arithmetic on
dequantized operands, rounded where the product rounds:
- fc1's input (the LN+modulate value) per row, the weights per output channel (tests/fp8_ref.py);
- fc2's input, the fp32 GELU output, per 1 x 128 block (no bf16 rounding in between: the fc1 epilogue emits the codes);
- in the single blocks, linear2's input cat(attn, gelu(mlp)) per 1 x 128 block: the bf16 attention output and the fp32
  GELU output.
`fp8_mlps()` patches the oracle module for the duration of a `with` block."""
import contextlib

import torch
import torch.nn.functional as F

from tests import fp8_ref as R


def qdq_blocks(x: torch.Tensor, block: int = 128) -> torch.Tensor:
    """fp32 [.., K] -> the dequantized e4m3 values with one scale per `block` columns."""
    shape = x.shape
    xb = x.float().reshape(*shape[:-1], shape[-1] // block, block)
    return R.dequantize(*R.quantize(xb)).reshape(shape)


def _lin(x, w, b):
    return x @ R.qdq(w.float()).t() + (0 if b is None else b.float())


def _mlp(x, W, pfx):
    h = F.gelu(_lin(R.qdq(x.float()), W[pfx + "0.weight"], W[pfx + "0.bias"]), approximate="tanh")
    return _lin(qdq_blocks(h), W[pfx + "2.weight"], W[pfx + "2.bias"]).to(x.dtype)


def _single_stream_block(M):
    def block(W, x, vec, pe, num_heads, fused_qkv):
        C = x.shape[-1]
        s, c, g = M.modulation(vec, W["modulation.lin.weight"], W["modulation.lin.bias"], 3)
        xm = M.ln_modulate(x, s, c)
        if fused_qkv:
            w1, b1 = W["linear1.weight"], W["linear1.bias"]
            wq, bq, wm, bm = w1[:3 * C], b1[:3 * C], w1[3 * C:], b1[3 * C:]
            q, k, v = F.linear(xm, wq, bq).chunk(3, dim=-1)
        else:
            q = F.linear(xm, W["q_proj.weight"], W["q_proj.bias"])
            k = F.linear(xm, W["k_proj.weight"], W["k_proj.bias"])
            v = F.linear(xm, W["v_mlp.weight"][:C], W["v_mlp.bias"][:C])
            wm, bm = W["v_mlp.weight"][C:], W["v_mlp.bias"][C:]
        q, k, v = M._heads(q, num_heads), M._heads(k, num_heads), M._heads(v, num_heads)
        q = M.rms_norm(q, W["norm.query_norm.scale"]).to(v)
        k = M.rms_norm(k, W["norm.key_norm.scale"]).to(v)
        a = M.attention(q, k, v, pe)
        h = F.gelu(_lin(R.qdq(xm.float()), wm, bm), approximate="tanh")
        out = _lin(qdq_blocks(torch.cat((a.float(), h), -1)), W["linear2.weight"], W["linear2.bias"]).to(x.dtype)
        return x + g * out
    return block


@contextlib.contextmanager
def fp8_mlps():
    """Patch oracle/mmdit_oracle.py so that `model_forward` runs every block MLP at the FP8 rounding points."""
    from oracle import mmdit_oracle as M

    saved = M._mlp, M.single_stream_block
    M._mlp, M.single_stream_block = _mlp, _single_stream_block(M)
    try:
        yield M
    finally:
        M._mlp, M.single_stream_block = saved
