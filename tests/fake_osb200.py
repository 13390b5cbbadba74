"""CPU stand-in for the `osb200` binding, used ONLY by the tests.

TEST INFRASTRUCTURE, not a fallback: the product never imports this module, and `osb200` itself still refuses to run
without CUDA.  The host side of the drop-in (opensora/models/*, utils/sampling.py) is a few thousand lines of shape /
stride / caching logic around the C ABI calls; this double implements the *documented contract* of every binding
function (include/osb200.h, open-sora_b200/osb200/__init__.py docstrings) with plain torch ops so that this logic can
be executed on the CPU box and compared with the oracle: patch embedding, modulation tables and `x_mask` indexing,
the packed kv projection, the row-stride conventions of spatial / temporal / cross attention, sequence-parallel
transpositions (gloo, world size 2), VAE padding / up-sampling / tiling arithmetic, the text encoders, LoRA / DoRA
and every FP8 mode.

One module defines each entry point once, in the binding's order and with the binding's signatures, so the `fake_osb`
fixture of tests/conftest.py installs the whole contract (`sys.modules["osb200"]` for the duration of one test).  The
GPU tests call some entries and helpers directly, on CUDA tensors too, to pin the stand-in to the kernels
(tests/test_double_conformance_gpu.py compares it element by element).

- Rounding points mirror the kernels: fp32 math, one rounding per op; RMSNorm rounds twice as T5LayerNorm does;
  attention rounds q-hat, k-hat and the unnormalised P to bf16.  Tolerances in the host tests are therefore the same
  bf16 noise floors as on the GPU.
- e4m3 quantization (the row, block and attention quantizers): s = amax / 448 per group (1 for an all-zero group),
  codes = the torch float8_e4m3fn cast of x / s (round to nearest even; |x / s| <= 448 by construction, the clamp only
  states the kernels' satfinite).
- Launches: one count per kernel launch in `launch_count()` and one (name, detail) entry in `calls`; a refused call
  counts nothing."""
import math

import torch
import torch.nn.functional as F

EPI_BIAS, EPI_BIAS_GELU_TANH, EPI_BIAS_GATE_RES = 0, 1, 2
EPI_GATED_GELU, EPI_BIAS_QUICK_GELU = 3, 4
EPI_BIAS_GELU_TANH_FP8 = 5
ATTN_IMPL = 0
ATTN_FP8_KEY_BLOCK = 128
E4M3 = torch.float8_e4m3fn
_launches = 0
calls = []   # (name, detail) log, so tests can assert how the host code drives the boundary

# Accumulation dtype of the bf16 GEMM, block-scaled FP8 GEMM and convolution stand-ins.  fp32 by default; a test that
# compares two decompositions of the SAME computation (e.g. a frame-sharded convolution against the whole one) switches
# to fp64, where the summation order of the CPU kernels can no longer flip a bf16 rounding, so the comparison can be
# bit-exact.  Read at call time: tests assign it.
ACC_DTYPE = torch.float32


class OsbError(RuntimeError):
    pass


def _count(name, detail=None, launches=1):
    global _launches
    _launches += launches
    calls.append((name, detail))


def reset():
    global _launches
    _launches = 0
    calls.clear()


def launch_count() -> int:
    return _launches


def init(device=None) -> None:
    pass


def start_profile():
    pass


def stop_profile():
    return []


def _need(t, dtype, name):
    if t is None:
        return
    if t.dtype != dtype:
        raise OsbError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() >= 1 and t.stride(-1) != 1 and t.shape[-1] != 1:
        raise OsbError(f"{name} must have unit stride in the last dimension")


def require_cuda_bf16(t, what: str) -> None:
    if t.dtype != torch.bfloat16:   # the dtype half of the contract still holds on the CPU double
        raise OsbError(f"{what} (osb200) runs in bfloat16 only")


def _put(val, out):
    """The result, or a copy into `out`; `out` may alias an input (in-place residual stream): `val` is materialised."""
    if out is None:
        return val
    out.copy_(val)
    return out


def _groups(rows, group_rows, mod_index, device):
    g = torch.arange(rows, device=device) // max(int(group_rows), 1)
    if mod_index is not None:
        g = mod_index.long()[g]
    return g


def _e4m3(x):
    return x.clamp(-448.0, 448.0).to(E4M3)


def _e4m3_scale(amax):
    """s = amax / 448, 1 for an all-zero group.  Divides by a tensor: on CUDA, torch divides by a Python scalar through
    its rounded reciprocal, which is not the kernels' division."""
    return torch.where(amax > 0, amax / torch.tensor(448.0, device=amax.device), torch.ones_like(amax))


class Scatter:
    def __init__(self, mode, P, rank, I, J, peers):
        self.mode, self.P, self.rank, self.I, self.J, self.peers = mode, P, rank, I, J, peers


def make_scatter(mode, P, rank, I, J, peer_bufs):
    """The double routes rows into torch tensors (`peer_bufs`) instead of raw pointers; only what one process can do on its
    own is supported: P == 1 (mode 3, the local transpose)."""
    return Scatter(mode, P, rank, I, J, peer_bufs)


def _ln_modulate(x, shift, scale, group_rows, mod_index, eps, fn, max_c):
    """The fp32 LayerNorm + modulate value of osb_ln_modulate(_fp8), before its rounding."""
    _need(x, torch.bfloat16, "x"); _need(shift, torch.float32, "shift"); _need(scale, torch.float32, "scale")
    _need(mod_index, torch.int32, "mod_index")
    assert x.dim() == 2 and x.is_contiguous()
    assert shift.dim() == 2 and scale.dim() == 2 and shift.stride(0) == scale.stride(0)
    rows, C = x.shape
    if C % 8 or C > max_c:
        raise OsbError(f"{fn} failed (-1): C must be a multiple of 8 and <= {max_c} (got {C})")
    xf = x.float()
    mu = xf.mean(-1, keepdim=True)
    var = (xf - mu).pow(2).mean(-1, keepdim=True)
    g = _groups(rows, group_rows, mod_index, x.device)
    return (xf - mu) * torch.rsqrt(var + eps) * (1.0 + scale[g]) + shift[g]


def ln_modulate(x, shift, scale, *, group_rows: int, mod_index=None, eps: float = 1e-6, out=None, scatter=None):
    if scatter is not None:
        assert scatter.mode == 3 and scatter.P == 1, "the CPU double only routes the local transpose"
        y = ln_modulate(x, shift, scale, group_rows=group_rows, mod_index=mod_index, eps=eps)
        I, J = scatter.I, scatter.J
        B = x.shape[0] // (I * J)
        scatter.peers[0].copy_(y.view(B, I, J, -1).transpose(1, 2).reshape(x.shape[0], -1))
        return None
    y = _ln_modulate(x, shift, scale, group_rows, mod_index, eps, "osb_ln_modulate", 8192).to(torch.bfloat16)
    _count("ln_modulate", tuple(x.shape))
    return _put(y, out)


def rms_norm(x, w, *, eps: float = 1e-6, out=None):
    _need(x, torch.bfloat16, "x"); _need(w, torch.bfloat16, "w")
    if x.dim() != 2 or not x.is_contiguous() or w.shape != (x.shape[1],):
        raise OsbError(f"rms_norm: x must be a contiguous [rows, C] tensor and w [C], got {tuple(x.shape)} and {tuple(w.shape)}")
    C = x.shape[1]
    if C % 8 or C > 4096:
        raise OsbError(f"osb_rms_norm failed (-1): osb_rms_norm: C must be a multiple of 8 and <= 4096 (got {C})")
    xf = x.float()
    t = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(torch.bfloat16)
    y = (w.float() * t.float()).to(torch.bfloat16)
    _count("rms_norm", tuple(x.shape))
    return _put(y, out)


# ---- GEMMs: one set of operand checks, one tail (bias, epilogue, one rounding, `out`); the accumulators differ --------
def _epilogue_shapes(fn, M, N, out_cols, out, bias, residual, gate, group_rows, mod_index):
    """The binding's extent checks of the optional GEMM operands (osb200._epilogue_shapes), raised before any math."""
    if out is not None and tuple(out.shape) != (M, out_cols):
        raise OsbError(f"{fn}: out must be [{M}, {out_cols}], got {tuple(out.shape)}")
    if bias is not None and tuple(bias.shape) != (N,):
        raise OsbError(f"{fn}: bias must be [{N}], got {tuple(bias.shape)}")
    if residual is not None and tuple(residual.shape) != (M, N):
        raise OsbError(f"{fn}: residual must be [{M}, {N}], got {tuple(residual.shape)}")
    groups = -(-M // (group_rows if group_rows > 0 else M))
    if gate is not None and (gate.dim() != 2 or gate.shape[1] != N or (mod_index is None and gate.shape[0] < groups)):
        raise OsbError(f"{fn}: gate must be [G, {N}] with G >= {groups} row groups, got {tuple(gate.shape)}")
    if mod_index is not None and (mod_index.dim() != 1 or mod_index.shape[0] < groups):
        raise OsbError(f"{fn}: mod_index must be 1-D with at least {groups} entries, got {tuple(mod_index.shape)}")


def _operands(fn, a, w, an, wn, dtype, bias, epilogue, residual, gate, group_rows, mod_index, out):
    """The checks every GEMM entry shares: dtypes, a [M, K] / w [N, K], the epilogue operands' extents.  (M, N, K)."""
    _need(a, dtype, an); _need(w, dtype, wn)
    for t, n in ((bias, "bias"), (residual, "residual")):
        _need(t, torch.bfloat16, n)
    _need(gate, torch.float32, "gate"); _need(mod_index, torch.int32, "mod_index")
    if a.dim() != 2 or w.dim() != 2 or a.shape[1] != w.shape[1]:
        raise OsbError(f"{fn}: {an} [M, K] and {wn} [N, K] expected, got {tuple(a.shape)} and {tuple(w.shape)}")
    M, K = a.shape
    N = w.shape[0]
    _epilogue_shapes(fn, M, N, N // 2 if epilogue == EPI_GATED_GELU else N, out, bias, residual, gate, group_rows,
                     mod_index)
    return M, N, K


def _gemm_args(fn, osb, a, w, bias, epilogue, residual, gate, group_rows, mod_index, out):
    """osb200._gemm_args and the refusals of the bf16 GEMM kernel (`osb` names it)."""
    M, N, K = _operands(fn, a, w, "a", "w", torch.bfloat16, bias, epilogue, residual, gate, group_rows, mod_index, out)
    _need(out, torch.bfloat16, "out")
    if not EPI_BIAS <= epilogue <= EPI_BIAS_QUICK_GELU:
        raise OsbError(f"{osb} failed (-1): {osb}: unknown epilogue {epilogue}")
    if K % 8 or N % 8:
        raise OsbError(f"{osb} failed (-1): {osb}: K and N must be multiples of 8 (K {K} N {N})")
    if (out.stride(0) if out is not None else N // 2 if epilogue == EPI_GATED_GELU else N) % 8:
        raise OsbError(f"{osb} failed (-1): {osb}: D must be 16-byte aligned with ldd % 8 == 0")
    return M, N, K


def _gemm_fp8_args(fn, a8, a_scale, w8, w_scale, bias, epilogue, residual, gate, group_rows, mod_index, out, out_scale,
                   block_n, blocks):
    """The checks of osb200.gemm_fp8 / _gemm_fp8_blocks and the refusals of the FP8 GEMM kernels.  `blocks`: a_scale
    may be [M, K / 128] and the FP8 GELU epilogue is built."""
    osb = "osb_" + fn
    _need(a_scale, torch.float32, "a_scale"); _need(w_scale, torch.float32, "w_scale")
    M, N, K = _operands(fn, a8, w8, "a8", "w8", E4M3, bias, epilogue, residual, gate, group_rows, mod_index, out)
    fp8_out = blocks and epilogue == EPI_BIAS_GELU_TANH_FP8
    _need(out, E4M3 if fp8_out else torch.bfloat16, "out")
    if K % 128:
        raise OsbError(f"{osb} failed (-1): {osb}: K must be a multiple of 128 (one e4m3 k-block), got {K}")
    if N % 8:
        raise OsbError(f"{osb} failed (-1): {osb}: N must be a multiple of 8, got {N}")
    scales = ((M,), (M, K // 128)) if blocks else ((M,),)
    if a_scale is None or w_scale is None or a_scale.shape not in scales or w_scale.shape != (N,):
        raise OsbError(f"{fn}: a_scale must be {' or '.join(str(list(s)) for s in scales)} and w_scale [{N}]")
    if fp8_out and out_scale is not None and tuple(out_scale.shape) != (M, N // 128):
        raise OsbError(f"out_scale must be a float32 [{M}, {N // 128}] tensor (row stride free)")
    if block_n not in ((0, 128) if fp8_out else (0, 64, 128)):
        raise OsbError(f"{osb} failed (-3): {osb}: unsupported block_n {block_n} (64 or 128)")
    if not (fp8_out or EPI_BIAS <= epilogue <= EPI_BIAS_GATE_RES):
        raise OsbError(f"{osb} failed (-1): {osb}: epilogue {epilogue} is not built for FP8")
    if fp8_out and N % 128:
        raise OsbError(f"{osb} failed (-1): {osb}: the FP8 GELU epilogue needs N % 128 == 0, got {N}")
    return M, N, K


def _lora_args(fn, M, N, u, b, col_scale, device):
    """The checks of a LoRA GEMM's update operands u [M, r], b [N, r] and DoRA's column scale; returns r."""
    _need(u, torch.bfloat16, "u"); _need(b, torch.bfloat16, "b")
    if u is None or b is None or u.dim() != 2 or b.dim() != 2 or u.shape[0] != M or b.shape[0] != N \
            or u.shape[1] != b.shape[1]:
        raise OsbError(f"{fn}: u must be [M, r] and b [N, r] for a {M} x {N} GEMM")
    if col_scale is not None and (col_scale.dtype != torch.float32 or col_scale.shape != (N,)
                                  or not col_scale.is_contiguous() or col_scale.device != device):
        raise OsbError(f"{fn}: col_scale must be a contiguous float32 [{N}] tensor on {device}")
    r = u.shape[1]
    if r <= 0 or r % 8:
        raise OsbError(f"osb_{fn} failed (-1): osb_{fn}: rank r must be a positive multiple of 8, got {r}")
    if u.stride(0) % 8 or b.stride(0) % 8:
        raise OsbError(f"osb_{fn} failed (-1): osb_{fn}: ldu and ldb must be multiples of 8")
    return r


def _epilogue(acc, bias, epilogue, residual, gate, group_rows, mod_index):
    """bias and the epilogue on the accumulator, in its dtype: the value the GEMM's one rounding is taken of."""
    dt = acc.dtype
    if bias is not None:
        acc = acc + bias.to(dt)
    if epilogue in (EPI_BIAS_GELU_TANH, EPI_BIAS_GELU_TANH_FP8):
        acc = F.gelu(acc, approximate="tanh")
    elif epilogue == EPI_BIAS_GATE_RES:
        if gate is not None:
            M = acc.shape[0]
            acc = acc * gate.to(dt)[_groups(M, group_rows if group_rows > 0 else M, mod_index, acc.device)]
        if residual is not None:
            acc = acc + residual.to(dt)
    elif epilogue == EPI_GATED_GELU:   # rows of w interleave wi_0 (even) and wi_1 (odd)
        acc = F.gelu(acc[:, 0::2], approximate="tanh") * acc[:, 1::2]
    elif epilogue == EPI_BIAS_QUICK_GELU:
        acc = acc * torch.sigmoid(1.702 * acc)
    return acc


def _store(y, epilogue, out, out_scale=None):
    """The GEMM's one rounding: to bf16, or for the FP8 GELU epilogue the 1 x 128 block rule ((codes, scales))."""
    if epilogue == EPI_BIAS_GELU_TANH_FP8:
        q, s = quant_blocks(y.float())
        return _put(q, out), _put(s, out_scale)
    return _put(y.to(torch.bfloat16), out)


def gemm(a, w, bias=None, *, epilogue: int = EPI_BIAS, residual=None, gate=None, group_rows: int = 0, mod_index=None,
         out=None, cta_group: int = 0, block_n: int = 0):
    M, N, K = _gemm_args("gemm", "osb_gemm_bf16", a, w, bias, epilogue, residual, gate, group_rows, mod_index, out)
    acc = a.to(ACC_DTYPE) @ w.to(ACC_DTYPE).t()
    _count("gemm", (M, N, K, epilogue))
    return _store(_epilogue(acc, bias, epilogue, residual, gate, group_rows, mod_index), epilogue, out)


def gemm_lora_fp32(a, w, bias, u, b, *, col_scale=None, epilogue=EPI_BIAS, residual=None, gate=None, group_rows=0,
                   mod_index=None, acc_dtype=torch.float32):
    """epilogue(col_scale * (a w^T + u b^T) + bias) before the rounding to bf16, accumulated in `acc_dtype`."""
    acc = a.to(acc_dtype) @ w.to(acc_dtype).t() + u.to(acc_dtype) @ b.to(acc_dtype).t()
    if col_scale is not None:
        acc = acc * col_scale.to(acc_dtype)
    return _epilogue(acc, bias, epilogue, residual, gate, group_rows, mod_index)


def gemm_lora(a, w, bias, u, b, *, epilogue: int = EPI_BIAS, residual=None, gate=None, group_rows: int = 0,
              mod_index=None, out=None, block_n: int = 0, col_scale=None):
    M, N, K = _gemm_args("gemm_lora", "osb_gemm_lora", a, w, bias, epilogue, residual, gate, group_rows, mod_index, out)
    r = _lora_args("gemm_lora", M, N, u, b, col_scale, a.device)
    y = gemm_lora_fp32(a, w, bias, u, b, col_scale=col_scale, epilogue=epilogue, residual=residual, gate=gate,
                       group_rows=group_rows, mod_index=mod_index, acc_dtype=ACC_DTYPE)
    _count("gemm_lora", (M, N, K, r, epilogue))
    return _store(y, epilogue, out)


def gemm_fp8(a8, a_scale, w8, w_scale, bias=None, *, epilogue: int = EPI_BIAS, residual=None, gate=None,
             group_rows: int = 0, mod_index=None, out=None, block_n: int = 0):
    M, N, K = _gemm_fp8_args("gemm_fp8", a8, a_scale, w8, w_scale, bias, epilogue, residual, gate, group_rows,
                             mod_index, out, None, block_n, blocks=False)
    acc = (a8.float() @ w8.float().t()) * (a_scale[:, None] * w_scale[None, :])   # fp32 whatever ACC_DTYPE is
    _count("gemm_fp8", (M, N, K, epilogue))
    return _store(_epilogue(acc, bias, epilogue, residual, gate, group_rows, mod_index), epilogue, out)


def ln_modulate_fp8(x, shift, scale, *, group_rows: int, mod_index=None, eps: float = 1e-6, out=None, out_scale=None):
    y = _ln_modulate(x, shift, scale, group_rows, mod_index, eps, "osb_ln_modulate_fp8", 4096)   # not rounded to bf16
    q, s = _quant(y)
    _count("ln_modulate_fp8", tuple(x.shape))
    return _put(q, out), _put(s, out_scale)


def quant_rows_fp8(x, *, out=None, out_scale=None):
    _need(x, torch.bfloat16, "x")
    if x.dim() != 2:
        raise OsbError(f"quant_rows_fp8: x must be [rows, K], got {tuple(x.shape)}")
    rows, K = x.shape
    if K % 8 or K > 8192:
        raise OsbError(f"osb_quant_rows_fp8 failed (-1): K must be a multiple of 8 and <= 8192 (got {K})")
    if x.stride(0) % 8:
        raise OsbError("osb_quant_rows_fp8 failed (-1): ldx must be a multiple of 8")
    q, s = _quant(x.float())
    _count("quant_rows_fp8", (rows, K))
    return _put(q, out), _put(s, out_scale)


def quant_blocks(x: torch.Tensor, block: int = 128):
    """fp32 [rows, K] -> (e4m3 codes [rows, K], fp32 scales [rows, K / block])."""
    rows, K = x.shape
    xb = x.float().reshape(rows, K // block, block)
    s = _e4m3_scale(xb.abs().amax(-1))
    return _e4m3(xb / s[..., None]).reshape(rows, K), s


def _quant(x):
    """fp32 rows -> (e4m3 codes, fp32 scales [rows]): the block rule with one block per row."""
    q, s = quant_blocks(x, x.shape[1])
    return q, s[:, 0]


def _fp8_blocks_acc(a8, a_scale, w8, w_scale, dt):
    """w_scale[n] * sum_kb a_scale[m, kb] * (the e4m3 products of 128-element k-block kb), accumulated in `dt`."""
    M, K = a8.shape
    KB = K // 128
    sa = a_scale.to(dt)[:, None].expand(M, KB) if a_scale.dim() == 1 else a_scale.to(dt)
    a, w = a8.to(dt), w8.to(dt)
    acc = torch.zeros(M, w8.shape[0], dtype=dt, device=a8.device)
    for kb in range(KB):
        k = slice(128 * kb, 128 * kb + 128)
        acc = acc + (a[:, k] @ w[:, k].t()) * sa[:, kb:kb + 1]
    return acc * w_scale.to(dt)


def gemm_fp8_blocks(a8, a_scale, w8, w_scale, bias=None, *, epilogue: int = EPI_BIAS, residual=None, gate=None,
                    group_rows: int = 0, mod_index=None, out=None, out_scale=None, block_n: int = 0):
    M, N, K = _gemm_fp8_args("gemm_fp8_blocks", a8, a_scale, w8, w_scale, bias, epilogue, residual, gate, group_rows,
                             mod_index, out, out_scale, block_n, blocks=True)
    acc = _fp8_blocks_acc(a8, a_scale, w8, w_scale, ACC_DTYPE)
    _count("gemm_fp8_blocks", (M, N, K, epilogue, a_scale.dim()))
    return _store(_epilogue(acc, bias, epilogue, residual, gate, group_rows, mod_index), epilogue, out, out_scale)


def gemm_fp8_lora_acc(a8, a_scale, w8, w_scale, u, b, col_scale=None, dt=torch.float32):
    """g * (w_scale * sum_kb a_scale[:, kb] * acc_kb + sum over 64-column tail blocks of u b^T), accumulated in `dt`:
    the rank tail is added unscaled, after w_scale, one 64-column k-block at a time."""
    acc = _fp8_blocks_acc(a8, a_scale, w8, w_scale, dt)
    uu, bb = u.to(dt), b.to(dt)
    for j0 in range(0, u.shape[1], 64):
        acc = acc + uu[:, j0:j0 + 64] @ bb[:, j0:j0 + 64].t()
    if col_scale is not None:
        acc = acc * col_scale.to(dt)
    return acc


def gemm_fp8_lora(a8, a_scale, w8, w_scale, bias, u, b, *, epilogue: int = EPI_BIAS, residual=None, gate=None,
                  group_rows: int = 0, mod_index=None, out=None, out_scale=None, block_n: int = 0, col_scale=None):
    M, N, K = _gemm_fp8_args("gemm_fp8_lora", a8, a_scale, w8, w_scale, bias, epilogue, residual, gate, group_rows,
                             mod_index, out, out_scale, block_n, blocks=True)
    r = _lora_args("gemm_fp8_lora", M, N, u, b, col_scale, a8.device)
    acc = gemm_fp8_lora_acc(a8, a_scale, w8, w_scale, u, b, col_scale, ACC_DTYPE)
    _count("gemm_fp8_lora", (M, N, K, r, epilogue, a_scale.dim()))
    return _store(_epilogue(acc, bias, epilogue, residual, gate, group_rows, mod_index), epilogue, out, out_scale)


def quant_blocks_fp8(x, *, block: int = 128, out=None, out_scale=None):
    _need(x, torch.bfloat16, "x")
    if x.dim() != 2:
        raise OsbError(f"quant_blocks_fp8: x must be [rows, K], got {tuple(x.shape)}")
    rows, K = x.shape
    if K % 128 or block not in (128, K):
        raise OsbError(f"osb_quant_blocks_fp8 failed (-1): K must be a positive multiple of 128 and block 128 or K "
                       f"(K {K} block {block})")
    if x.stride(0) % 8:
        raise OsbError("osb_quant_blocks_fp8 failed (-1): ldx must be a multiple of 8")
    q, s = quant_blocks(x, block)
    _count("quant_blocks_fp8", (rows, K, block))
    return _put(q, out), _put(s, out_scale)


def interleave_gated(wi_0, wi_1):
    return torch.stack((wi_0, wi_1), dim=1).reshape(2 * wi_0.shape[0], wi_0.shape[1]).contiguous()


# ---- attention: one staging (rows, QK-RMSNorm, RoPE, bf16 q-hat / k-hat) for attn_short, attn_short_bias and the FP8
# attention ---------------------------------------------------------------------------------------------------------
def _rms(x, w, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def _rope_interleaved(x, cos, sin):   # x [..., L, D], tables [L, D/2]: pairs (2i, 2i+1)
    x1, x2 = x[..., 0::2], x[..., 1::2]
    return torch.stack((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1).flatten(-2)


def _rope_half(x, cos, sin):          # pairs (i, i + D/2)
    h = x.shape[-1] // 2
    x1, x2 = x[..., :h], x[..., h:]
    return torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1)


def _pairs(who, q_norm_w, k_norm_w, rope_cos, rope_sin, q_norm_w2, k_norm_w2):
    if (q_norm_w is None) != (k_norm_w is None) or (rope_cos is None) != (rope_sin is None):
        raise OsbError(f"{who}: norm weights / rope tables must come in pairs")
    if (q_norm_w2 is None) != (k_norm_w2 is None) or (q_norm_w2 is not None and q_norm_w is None):
        raise OsbError(f"{who}: the second norm weight pair needs the first")


def stage(q, k, v, *, num_seqs, q_strides, k_strides, L, H, q_norm_w=None, k_norm_w=None, norm_eps=1e-6, rope_cos=None,
          rope_sin=None, q_norm_w2=None, k_norm_w2=None, norm_split=0, rope_half=False, seqs_per_batch=1, Lk=None,
          D=128):
    """(q~, k~, v) as fp32 [num_seqs, H, L, D] (k and v with Lk tokens, default L) and the [num_seqs, L] query rows, as
    osb_attn_short stages them: token t of sequence s = (b, j) is row b * batch_stride + j * seq_stride + t * tok_stride;
    fp32 RMSNorm with the stream's weight (the second pair from token norm_split on), RoPE by position, one rounding of
    q~ and k~ to bf16."""
    Lk = L if Lk is None else Lk
    dev = q.device
    s = torch.arange(num_seqs, device=dev)
    b, j = s // seqs_per_batch, s % seqs_per_batch

    def rows(strides, n):
        bs, ss, ts = strides
        return (b * bs + j * ss)[:, None] + torch.arange(n, device=dev)[None] * ts

    def gather(x, r, n):
        return x[r][..., : H * D].float().view(num_seqs, n, H, D).transpose(1, 2)

    rq, rk = rows(q_strides, L), rows(k_strides, Lk)
    qf, kf, vf = gather(q, rq, L), gather(k, rk, Lk), gather(v, rk, Lk)
    if q_norm_w is not None:
        def normed(x, w, w2, n):
            y = _rms(x, w.float(), norm_eps)
            if w2 is not None:
                sel = (torch.arange(n, device=dev) >= norm_split)[None, None, :, None]
                y = torch.where(sel, _rms(x, w2.float(), norm_eps), y)
            return y
        qf, kf = normed(qf, q_norm_w, q_norm_w2, L), normed(kf, k_norm_w, k_norm_w2, Lk)
    if rope_cos is not None:
        rot = _rope_half if rope_half else _rope_interleaved
        qf, kf = rot(qf, rope_cos[:L], rope_sin[:L]), rot(kf, rope_cos[:Lk], rope_sin[:Lk])
    return qf.to(torch.bfloat16).float(), kf.to(torch.bfloat16).float(), vf, rq


def _token_rows(o):
    """[n, H, L, D] -> [n * L, H * D]: one row per token, heads side by side."""
    n, H, L, D = o.shape
    return o.transpose(1, 2).reshape(n * L, H * D)


def _softmax_pv(sc, vf, kv_lens):
    """softmax(sc) V with keys past kv_lens masked: the unnormalised P is rounded to bf16 before P V, the row sum is
    taken over the unrounded P, a row with no visible key is zero."""
    if kv_lens is not None:
        dead = torch.arange(sc.shape[-1], device=sc.device)[None, :] >= kv_lens.long()[:, None]
        sc = sc.masked_fill(dead[:, None, None, :], float("-inf"))
    m = sc.amax(-1, keepdim=True)
    p = torch.exp(sc - torch.where(torch.isinf(m), torch.zeros_like(m), m))
    l = p.sum(-1, keepdim=True)
    return (p.to(torch.bfloat16).float() @ vf) / torch.where(l > 0, l, torch.ones_like(l))


def attn_short(q, k, v, out, *, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int, num_heads: int,
               head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None, norm_eps: float = 1e-6, rope_cos=None,
               rope_sin=None, softmax_scale=None, q_norm_w2=None, k_norm_w2=None, norm_split: int = 0, impl: int = 0,
               rope_half: bool = False):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out"), (q_norm_w, "q_norm_w"), (k_norm_w, "k_norm_w")):
        _need(t, torch.bfloat16, n)
    _need(rope_cos, torch.float32, "rope_cos"); _need(rope_sin, torch.float32, "rope_sin"); _need(kv_lens, torch.int32, "kv_lens")
    _pairs("osb_attn_short", q_norm_w, k_norm_w, rope_cos, rope_sin, q_norm_w2, k_norm_w2)
    H, D = num_heads, head_dim
    if D not in (64, 72, 128):
        raise OsbError(f"osb_attn_short failed (-1): head_dim {D} not built (64, 72, 128)")
    if rope_cos is not None and rope_half and D % 16:
        raise OsbError("osb_attn_short failed (-1): rotate-half RoPE needs head_dim % 16 == 0")
    qf, kf, vf, rq = stage(q, k, v, num_seqs=num_seqs, seqs_per_batch=seqs_per_batch, q_strides=q_strides,
                           k_strides=k_strides, L=Lq, Lk=Lk, H=H, D=D, q_norm_w=q_norm_w, k_norm_w=k_norm_w,
                           norm_eps=norm_eps, rope_cos=rope_cos, rope_sin=rope_sin, q_norm_w2=q_norm_w2,
                           k_norm_w2=k_norm_w2, norm_split=norm_split, rope_half=rope_half)
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    o = _softmax_pv((qf @ kf.transpose(-1, -2)) * scale, vf, kv_lens)
    out[rq.reshape(-1), : H * D] = _token_rows(o).to(torch.bfloat16)
    _count("attn_short", (num_seqs, Lq, Lk, H, D))
    return out


def attn_short_bias(q, k, v, out, bias, *, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int,
                    num_heads: int, head_dim: int, kv_lens=None, softmax_scale=None):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        _need(t, torch.bfloat16, n)
    _need(bias, torch.float32, "bias"); _need(kv_lens, torch.int32, "kv_lens")
    H, D = num_heads, head_dim
    n_rel = Lq + Lk - 1
    if bias is None or not bias.is_contiguous() or bias.shape not in ((n_rel,), (H, n_rel)):
        raise OsbError(f"attn_short_bias: bias must be a contiguous fp32 [{n_rel}] or [{H}, {n_rel}] tensor, got "
                       f"{None if bias is None else tuple(bias.shape)}")
    if D != 64:
        raise OsbError(f"osb_attn_short_bias failed (-1): osb_attn_short_bias: head_dim {D} not built (64)")
    qf, kf, vf, rq = stage(q, k, v, num_seqs=num_seqs, seqs_per_batch=seqs_per_batch, q_strides=q_strides,
                           k_strides=k_strides, L=Lq, Lk=Lk, H=H, D=D)
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    rel = torch.arange(Lk, device=q.device)[None, :] - torch.arange(Lq, device=q.device)[:, None] + Lq - 1
    bb = bias.view(-1, n_rel)[:, rel]                                               # [1 or H, Lq, Lk]
    o = _softmax_pv((qf @ kf.transpose(-1, -2)) * scale + bb[None], vf, kv_lens)
    out[rq.reshape(-1), : H * D] = _token_rows(o).to(torch.bfloat16)
    _count("attn_short", (num_seqs, Lq, Lk, H, D, "bias"))
    return out


def visible_keys(Lq: int, Lk: int, frame_tokens: int, q_frame0: int, device) -> torch.Tensor:
    """[Lq] number of keys each query token sees: min(Lk, (q_frame0 + i // frame_tokens + 1) * frame_tokens)."""
    i = torch.arange(Lq, device=device)
    return torch.clamp((q_frame0 + i // frame_tokens + 1) * frame_tokens, max=Lk)


def attn_frames(q, k, v, *, frame_tokens: int, q_frame0: int = 0, out=None, softmax_scale=None):
    """Frame-causal attention as osb_attn_frames computes it: fp32 scores, exact softmax with the row maximum over the
    visible keys, P rounded to bf16 unnormalised before P V, the row sum from the unrounded P, one rounding."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        _need(t, torch.bfloat16, n)
    if q.dim() != 3 or k.dim() != 3 or k.shape != v.shape or q.shape[0] != k.shape[0] or q.shape[2] != k.shape[2]:
        raise OsbError(f"attn_frames: q [batch, Lq, D] and k, v [batch, Lk, D] expected, got {tuple(q.shape)}, "
                       f"{tuple(k.shape)}, {tuple(v.shape)}")
    nb, Lq, D = q.shape
    Lk = k.shape[1]
    if out is not None and out.shape != q.shape:
        raise OsbError(f"attn_frames: out must have q's shape {tuple(q.shape)}, got {tuple(out.shape)}")
    if nb > 1 and (k.stride(0) * v.stride(1) != v.stride(0) * k.stride(1)):
        raise OsbError("attn_frames: v must have k's batch stride and out q's (in rows)")
    fail = "osb_attn_frames failed (-1): osb_attn_frames: "
    if D != 512:
        raise OsbError(fail + f"head_dim {D} not built (512)")
    lds = [t.stride(1) if t.shape[1] > 1 else max(t.stride(1), D) for t in (q, k, v)]
    if any(ld < 512 or ld % 8 for ld in lds):
        raise OsbError(fail + "leading dimensions must be >= 512 and multiples of 8")
    if frame_tokens < 1:
        raise OsbError(fail + f"frame_tokens must be >= 1, got {frame_tokens}")
    if Lq < 1:
        raise OsbError(fail + f"empty problem (batch {nb}, Lq {Lq})")
    if q_frame0 < 0 or Lk < 1:
        raise OsbError(fail + f"a query would see no key (q_frame0 {q_frame0}, Lk {Lk})")
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    sc = (q.float() @ k.float().transpose(1, 2)) * scale
    dead = torch.arange(Lk, device=q.device)[None, :] >= visible_keys(Lq, Lk, frame_tokens, q_frame0, q.device)[:, None]
    sc = sc.masked_fill(dead[None], float("-inf"))
    p = torch.exp(sc - sc.amax(-1, keepdim=True))          # every row sees key 0
    o = ((p.to(torch.bfloat16).float() @ v.float()) / p.sum(-1, keepdim=True)).to(torch.bfloat16)
    _count("attn_frames", (nb, Lq, Lk, D, frame_tokens, q_frame0))
    return _put(o, out)


# ---- FP8 attention (osb_attn_fp8): the workspace in the header's layout - q8 / k8 [B*H, Lpad, 128] with zero codes and
# scale 1 past L, per (token, head) scales; vt8 [B*H, 128, Lpad] with key vt8_key(p) at position p, per channel scales
# over the sequence.  Attention from the workspace operands as the kernel computes it: key blocks of 128, scores in log2
# units, online maximum, P8 = e4m3(256 p), partial P8 V8 promoted as O = alpha O + partial, out = O s_v / (256 l). -----
def vt8_key(pos: torch.Tensor) -> torch.Tensor:
    """Key held at position `pos` of vt8 (include/osb200.h): j(p) = 16 (p/16) + 2 ((p%16)/4) + p%2 + 8 ((p%4)/2) inside
    each 32-key group."""
    return (pos & ~31) + 16 * ((pos >> 4) & 1) + 2 * ((pos >> 2) & 3) + (pos & 1) + 8 * ((pos >> 1) & 1)


class AttnFp8Workspace:
    def __init__(self, B: int, L: int, H: int, device):
        BH, Lp = B * H, -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
        self.B, self.L, self.H, self.Lpad = B, L, H, Lp
        self.q8 = torch.empty(BH, Lp, 128, dtype=E4M3, device=device)
        self.k8 = torch.empty(BH, Lp, 128, dtype=E4M3, device=device)
        self.vt8 = torch.empty(BH, 128, Lp, dtype=E4M3, device=device)
        self.s_q = torch.empty(BH, Lp, device=device)
        self.s_k = torch.empty(BH, Lp, device=device)
        self.s_v = torch.empty(BH, 128, device=device)
        self.v_amax = torch.zeros(BH, 128, device=device)


def attn_fp8_workspace(B: int, L: int, H: int, device) -> AttnFp8Workspace:
    return AttnFp8Workspace(B, L, H, device)


def fill_workspace(ws: AttnFp8Workspace, qf, kf, vf) -> None:
    """Quantize staged [n, H, L, 128] operands into `ws` in the header's layout."""
    n, H, L, D = qf.shape
    BH, Lp = n * H, -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
    views = dict(q8=(BH, Lp, D), k8=(BH, Lp, D), vt8=(BH, D, Lp), s_q=(BH, Lp), s_k=(BH, Lp), s_v=(BH, D))
    t = {name: getattr(ws, name).view(-1)[:math.prod(shape)].view(shape) for name, shape in views.items()}
    for name, x in (("q", qf), ("k", kf)):
        s = _e4m3_scale(x.abs().amax(-1)).reshape(BH, L)
        codes = _e4m3(x.reshape(BH, L, D) / s[..., None])
        t[name + "8"].zero_()
        t[name + "8"][:, :L] = codes
        t["s_" + name].fill_(1.0)
        t["s_" + name][:, :L] = s
    sv = _e4m3_scale(vf.abs().amax(2)).reshape(BH, D)
    v8 = torch.zeros(BH, Lp, D, dtype=E4M3, device=vf.device)
    v8[:, :L] = _e4m3(vf.reshape(BH, L, D) / sv[:, None, :])
    t["s_v"].copy_(sv)
    t["vt8"].copy_(v8[:, vt8_key(torch.arange(Lp, device=vf.device))].transpose(1, 2))


def workspace_operands(ws: AttnFp8Workspace, BH: int, L: int):
    """(q8, s_q, k8, s_k, v8 in key order, s_v) of the first BH sequence-heads, read back from the workspace."""
    Lp = -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
    q8 = ws.q8.view(-1)[:BH * Lp * 128].view(BH, Lp, 128)
    k8 = ws.k8.view(-1)[:BH * Lp * 128].view(BH, Lp, 128)
    vt8 = ws.vt8.view(-1)[:BH * 128 * Lp].view(BH, 128, Lp)
    v8 = torch.empty(BH, Lp, 128, dtype=E4M3, device=vt8.device)
    v8[:, vt8_key(torch.arange(Lp, device=vt8.device))] = vt8.transpose(1, 2)
    return (q8, ws.s_q.view(-1)[:BH * Lp].view(BH, Lp), k8, ws.s_k.view(-1)[:BH * Lp].view(BH, Lp), v8,
            ws.s_v.view(-1)[:BH * 128].view(BH, 128))


def attention_from_workspace(ws: AttnFp8Workspace, BH: int, L: int, softmax_scale: float) -> torch.Tensor:
    """fp32 [BH, L, 128] output of the contract's online FP8 attention, from the workspace operands."""
    q8, sq, k8, sk, v8, sv = workspace_operands(ws, BH, L)
    sc = softmax_scale * 1.4426950408889634
    qd, kd, vd = q8[:, :L].float(), k8.float(), v8.float()
    m = torch.full((BH, L, 1), float("-inf"), device=q8.device)
    l = torch.zeros(BH, L, 1, device=q8.device)
    o = torch.zeros(BH, L, 128, device=q8.device)
    for k0 in range(0, L, ATTN_FP8_KEY_BLOCK):
        blk = slice(k0, k0 + ATTN_FP8_KEY_BLOCK)
        s = (qd @ kd[:, blk].transpose(1, 2)) * (sq[:, :L, None] * sc) * sk[:, None, blk]
        s = s.masked_fill(torch.arange(k0, k0 + ATTN_FP8_KEY_BLOCK, device=q8.device) >= L, float("-inf"))
        mn = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp2(m - mn)
        p = torch.exp2(s - mn)
        l = l * alpha + p.sum(-1, keepdim=True)
        o = o * alpha + _e4m3(256.0 * p).float() @ vd[:, blk]
        m = mn
    return o * sv[:, None, :] / (256.0 * l)


def _attn_fp8(fn, q, k, v, *, workspace, num_seqs, seqs_per_batch, q_strides, k_strides, Lq, Lk, num_heads, head_dim,
              kv_lens, q_norm_w, k_norm_w, norm_eps, rope_cos, rope_sin, softmax_scale, q_norm_w2, k_norm_w2,
              norm_split, impl, rope_half):
    """The refusals of osb_attn_fp8 / osb_attn_fp8_blocks, then stage, quantize into the workspace and attend: the fp32
    output [num_seqs * Lq, H * 128] and its rows of `out`."""
    fail = f"osb_{fn} failed (-1)"
    if head_dim != 128:
        raise OsbError(f"{fail}: osb_{fn}: head_dim {head_dim} not built (128)")
    if Lq != Lk:
        raise OsbError(f"{fail}: osb_{fn}: self-attention only (Lq {Lq} != Lk {Lk})")
    if kv_lens is not None:
        raise OsbError(f"{fail}: osb_{fn}: kv_lens is not supported")
    if seqs_per_batch != 1:
        raise OsbError(f"{fail}: osb_{fn}: one sequence per batch element")
    _pairs(fail, q_norm_w, k_norm_w, rope_cos, rope_sin, q_norm_w2, k_norm_w2)
    if not isinstance(workspace, AttnFp8Workspace):
        raise OsbError(f"{fn}: workspace must come from attn_fp8_workspace()")
    L, H = Lq, num_heads
    if num_seqs * H > workspace.s_v.shape[0] or -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK > workspace.Lpad:
        raise OsbError(f"{fail}: workspace too small")
    qf, kf, vf, rq = stage(q, k, v, num_seqs=num_seqs, q_strides=q_strides, k_strides=k_strides, L=L, H=H,
                           q_norm_w=q_norm_w, k_norm_w=k_norm_w, norm_eps=norm_eps, rope_cos=rope_cos, rope_sin=rope_sin,
                           q_norm_w2=q_norm_w2, k_norm_w2=k_norm_w2, norm_split=norm_split, rope_half=rope_half)
    fill_workspace(workspace, qf, kf, vf)
    scale = softmax_scale if softmax_scale is not None else head_dim ** -0.5
    o = attention_from_workspace(workspace, num_seqs * H, L, scale)
    return _token_rows(o.view(num_seqs, H, L, 128)), rq.reshape(-1)


def attn_fp8(q, k, v, out, *, workspace, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int,
             num_heads: int, head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None, norm_eps: float = 1e-6,
             rope_cos=None, rope_sin=None, softmax_scale=None, q_norm_w2=None, k_norm_w2=None, norm_split: int = 0,
             impl: int = 0, rope_half: bool = False):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out"), (q_norm_w, "q_norm_w"), (k_norm_w, "k_norm_w")):
        _need(t, torch.bfloat16, n)
    _need(rope_cos, torch.float32, "rope_cos"); _need(rope_sin, torch.float32, "rope_sin")
    o, rows = _attn_fp8("attn_fp8", q, k, v, workspace=workspace, num_seqs=num_seqs, seqs_per_batch=seqs_per_batch,
                        q_strides=q_strides, k_strides=k_strides, Lq=Lq, Lk=Lk, num_heads=num_heads, head_dim=head_dim,
                        kv_lens=kv_lens, q_norm_w=q_norm_w, k_norm_w=k_norm_w, norm_eps=norm_eps, rope_cos=rope_cos,
                        rope_sin=rope_sin, softmax_scale=softmax_scale, q_norm_w2=q_norm_w2, k_norm_w2=k_norm_w2,
                        norm_split=norm_split, impl=impl, rope_half=rope_half)
    out[rows, : num_heads * 128] = o.to(torch.bfloat16)
    _count("attn_fp8", (num_seqs, Lq, num_heads), launches=3)
    return out


def attn_fp8_blocks(q, k, v, out, out_scale, *, workspace, num_seqs: int, seqs_per_batch: int, q_strides, k_strides,
                    Lq: int, Lk: int, num_heads: int, head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None,
                    norm_eps: float = 1e-6, rope_cos=None, rope_sin=None, softmax_scale=None, q_norm_w2=None,
                    k_norm_w2=None, norm_split: int = 0, impl: int = 0, rope_half: bool = False):
    """`attn_fp8` up to the fp32 value v = O s_v / (256 l); each (row, head) of v is then one 1 x 128 block of the block
    rule.  Codes and scales go to column slices with a free row stride."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (q_norm_w, "q_norm_w"), (k_norm_w, "k_norm_w")):
        _need(t, torch.bfloat16, n)
    _need(out, E4M3, "out"); _need(out_scale, torch.float32, "out_scale")
    _need(rope_cos, torch.float32, "rope_cos"); _need(rope_sin, torch.float32, "rope_sin")
    for t, n, w in ((out, "out", num_heads * head_dim), (out_scale, "out_scale", num_heads)):
        if t is None or t.dim() != 2 or t.stride(1) != 1 or t.shape[1] < w:
            raise OsbError(f"attn_fp8_blocks: {n} must be a 2-D tensor of >= {w} unit-stride columns")
    if out.stride(0) % 8:
        raise OsbError("osb_attn_fp8_blocks failed (-1): leading dimensions must be multiples of 8 elements")
    o, rows = _attn_fp8("attn_fp8_blocks", q, k, v, workspace=workspace, num_seqs=num_seqs,
                        seqs_per_batch=seqs_per_batch, q_strides=q_strides, k_strides=k_strides, Lq=Lq, Lk=Lk,
                        num_heads=num_heads, head_dim=head_dim, kv_lens=kv_lens, q_norm_w=q_norm_w, k_norm_w=k_norm_w,
                        norm_eps=norm_eps, rope_cos=rope_cos, rope_sin=rope_sin, softmax_scale=softmax_scale,
                        q_norm_w2=q_norm_w2, k_norm_w2=k_norm_w2, norm_split=norm_split, impl=impl, rope_half=rope_half)
    codes, s = quant_blocks(o)
    out[rows, : num_heads * 128] = codes
    out_scale[rows, :num_heads] = s
    _count("attn_fp8_blocks", (num_seqs, Lq, num_heads), launches=3)
    return out, out_scale


# ---- head tiles (include/osb200.h osb_gemm_head_tiles / osb_attn_tiles): the double keeps the tile buffer as a dense
# [kinds, rows, heads*D] tensor - the byte layout of a tile is the kernels' business, the CONTRACT is which token row and
# head a value belongs to, what was applied to it (bias, RMSNorm, RoPE by position) and which keys a query may see. ------
# The tile map is host arithmetic of the binding itself (pure Python over a ctypes struct, no device needed): the double
# uses it as is, so the two can never disagree on how a sequence is tiled.
from osb200 import TileMap, tile_map  # noqa: E402,F401


class HeadTiles:
    def __init__(self, rows, tmap, kinds, heads, head_dim, device):
        if tmap.mode == 0:
            assert rows % tmap.L == 0, "rows must be whole sequences"
        else:
            assert tmap.T == tmap.L and tmap.S > 0 and rows % (tmap.S * tmap.T) == 0
        self.rows, self.map, self.kinds, self.heads, self.head_dim = rows, tmap, kinds, heads, head_dim
        self.dense = torch.zeros(kinds, rows, heads * head_dim, dtype=torch.bfloat16, device=device)


def _seq_pos(m, rows, device):
    r = torch.arange(rows, device=device)
    if m.mode == 0:
        return r // m.L, r % m.L
    b, rem = r // (m.T * m.S), r % (m.T * m.S)
    return b * m.S + rem % m.S, rem // m.S


def gemm_head_tiles(a, w, bias, tiles, *, nkinds, norm_w=(), rope=None, rope_kinds=0, eps=1e-6, kind0=0, general=False):
    for t, n in ((a, "a"), (w, "w"), (bias, "bias")):
        _need(t, torch.bfloat16, n)
    M, K = a.shape
    N = w.shape[0]
    H, D = tiles.heads, tiles.head_dim
    Cc = H * D
    assert M == tiles.rows and N % Cc == 0 and kind0 + N // Cc <= tiles.kinds and a.shape[1] == w.shape[1]
    if D not in (64, 72, 128) or H % 2:
        raise OsbError("osb_gemm_head_tiles failed (-1): head_dim / head count not built")
    if K % 8:
        raise OsbError(f"osb_gemm_head_tiles failed (-1): K must be a multiple of 8 (K {K})")
    if not 1 <= nkinds <= 4:
        raise OsbError(f"osb_gemm_head_tiles failed (-1): nkinds must be 1..4, got {nkinds}")
    if any(nw is not None for nw in norm_w[nkinds:]):
        raise OsbError("osb_gemm_head_tiles failed (-1): RMSNorm weight given for a kind >= nkinds")
    acc = a.float() @ w.float().t()
    if bias is not None:
        acc = acc + bias.float()
    _, pos = _seq_pos(tiles.map, M, a.device)
    for kidx in range(N // Cc):
        kind = kidx % nkinds
        x = acc[:, kidx * Cc:(kidx + 1) * Cc].reshape(M, H, D)
        nw = norm_w[kind] if kind < len(norm_w) else None
        if nw is not None:
            x = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * nw.float()
        if rope is not None and (rope_kinds >> kind) & 1:
            c, s_ = rope[0][pos][:, None, :], rope[1][pos][:, None, :]
            xa, xb = x[..., 0::2], x[..., 1::2]
            x = torch.stack((xa * c - xb * s_, xb * c + xa * s_), dim=-1).reshape(M, H, D)
        tiles.dense[kind0 + kidx] = x.reshape(M, Cc).to(torch.bfloat16)
    _count("gemm", (M, N, K, "head_tiles"))
    return tiles


def attn_tiles(q, kv, out, *, q_kind=0, k_kind=1, v_kind=2, Lk, num_seqs, kv_lens=None, softmax_scale=None,
               out_scatter=None, out_ld=None, out_map=None):
    H, D = q.heads, q.head_dim
    m = q.map
    if kv_lens is not None and m.G > 1:
        raise OsbError("attn_tiles: kv_lens applies to unpacked query maps only (G == 1); packed sequences see all Lk keys")
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    seq_q, pos_q = _seq_pos(m, q.rows, out.device)
    out_rows = None
    if out_map is not None:   # output rows in another token order: (seq, pos) -> row of `out`
        assert out_map.key()[4:] == m.key()[4:] and out_map.L == m.L
        so, po = _seq_pos(out_map, q.rows, out.device)
        inv = torch.empty(q.rows, dtype=torch.long, device=out.device)
        inv[so * m.L + po] = torch.arange(q.rows, device=out.device)
        out_rows = inv[seq_q * m.L + pos_q]
    seq_k, pos_k = _seq_pos(kv.map, kv.rows, out.device)
    assert int(seq_q.max()) + 1 == num_seqs
    for s in range(num_seqs):
        rq = (seq_q == s).nonzero().flatten()
        rk = (seq_k == s).nonzero().flatten()
        rk = rk[pos_k[rk].argsort()]
        n = Lk if kv_lens is None else min(int(kv_lens[s]), Lk)
        ro = rq if out_rows is None else out_rows[rq]
        if n <= 0:
            out[ro] = 0
            continue
        rk = rk[:n]
        qq = q.dense[q_kind][rq].float().view(-1, H, D).permute(1, 0, 2)
        kk = kv.dense[k_kind][rk].float().view(-1, H, D).permute(1, 0, 2)
        vv = kv.dense[v_kind][rk].float().view(-1, H, D).permute(1, 0, 2)
        sc = qq @ kk.transpose(-1, -2) * scale
        p = torch.exp(sc - sc.amax(-1, keepdim=True))
        # as the kernel: the UNnormalised P is rounded to bf16 for P V, the sum is taken over the unrounded P
        o = (p.to(torch.bfloat16).float() @ vv) / p.sum(-1, keepdim=True)
        out[ro] = o.permute(1, 0, 2).reshape(len(rq), H * D).to(torch.bfloat16)
    _count("attn_tiles", (num_seqs, m.L, Lk, H, D))
    return out


# ---- FP8 head tiles (osb_head_tiles_fp8 / osb_attn_tiles_fp8), kept in their logical layout (the 128-byte swizzle of the
# real buffer is the kernels' business): `codes` e4m3 [kinds, heads, tiles, 128, 128] (q / k: [tile row][channel]; v:
# [channel][position p], holding key vt8_key(p) of the tile) and `scales` fp32 [kinds, heads, tiles, 128].  Tiles are
# filled from the dense rows of HeadTiles through the binding's tile map, so rows no token maps to are zero, as in the
# real buffer.  Attention from those operands as the kernel computes it: key tiles in order, scores in log2 units,
# online maximum, P8 = e4m3(256 p), partial P8 V8 promoted as O = alpha O + s_v (.) partial, out = O / (256 l). -------
def tile_index(m, rows: int, device):
    """(tile, row in tile) of every token row under tile map `m` (tiles.cuh tile_of_row)."""
    seq, pos = _seq_pos(m, rows, device)
    if m.G > 1:
        return seq // m.G, (seq % m.G) * m.L + pos
    return seq * m.tps + pos // m.tile_rows, pos % m.tile_rows


def tiles_per_head(m, rows: int) -> int:
    seqs = rows // m.L
    return -(-seqs // m.G) if m.G > 1 else seqs * m.tps


class HeadTilesFp8:
    def __init__(self, tiles):
        if tiles.head_dim not in (64, 72):
            raise OsbError(f"FP8 head tiles are built for head_dim 64 and 72, not {tiles.head_dim}")
        self.src, self.map, self.kinds, self.heads, self.head_dim = tiles, tiles.map, tiles.kinds, tiles.heads, tiles.head_dim
        self.rows = tiles.rows
        self.tiles_per_head = tiles_per_head(tiles.map, tiles.rows)
        dev = tiles.dense.device
        self.codes = torch.zeros(self.kinds, self.heads, self.tiles_per_head, 128, 128, dtype=E4M3, device=dev)
        self.scales = torch.zeros(self.kinds, self.heads, self.tiles_per_head, 128, device=dev)


def bf16_tiles(tiles, kind: int) -> torch.Tensor:
    """fp32 [heads, tiles, 128, D]: the bf16 head tiles of one kind, rows past a tile's end zero."""
    H, D, dev = tiles.heads, tiles.head_dim, tiles.dense.device
    t, r = tile_index(tiles.map, tiles.rows, dev)
    x = torch.zeros(H, tiles_per_head(tiles.map, tiles.rows), 128, D, device=dev)
    x[:, t, r] = tiles.dense[kind].float().view(-1, H, D).transpose(0, 1)
    return x


def convert_qk(x: torch.Tensor):
    """[.., 128, D] fp32 -> (codes [.., 128, 128] e4m3, scales [.., 128]): per row."""
    s = _e4m3_scale(x.abs().amax(-1))
    codes = torch.zeros(*x.shape[:-1], 128, dtype=E4M3, device=x.device)
    codes[..., : x.shape[-1]] = _e4m3(x / s[..., None])
    return codes, s


def convert_v(x: torch.Tensor):
    """[.., 128 keys, D] fp32 -> (codes [.., 128 channels, 128 positions] e4m3, scales [.., 128]): per channel over the
    tile, positions in the vt8 key order; channels past D zero with scale 1."""
    D = x.shape[-1]
    s = torch.ones(*x.shape[:-2], 128, device=x.device)
    s[..., :D] = _e4m3_scale(x.abs().amax(-2))
    codes = torch.zeros(*x.shape[:-2], 128, 128, dtype=E4M3, device=x.device)
    keys = vt8_key(torch.arange(128, device=x.device))
    codes[..., :D, :] = _e4m3(x[..., keys, :] / s[..., None, :D]).transpose(-1, -2)
    return codes, s


def head_tiles_fp8(tiles, dst, *, kind0: int = 0, nkinds=None, v_period: int = 0, v_slot: int = 0):
    if dst.src is not tiles:
        raise OsbError("head_tiles_fp8: dst must be HeadTilesFp8(tiles) of the same bf16 tiles")
    nkinds = tiles.kinds - kind0 if nkinds is None else nkinds
    if not (0 <= kind0 and nkinds >= 1 and kind0 + nkinds <= tiles.kinds):
        raise OsbError(f"head_tiles_fp8: kinds [{kind0}, {kind0 + nkinds}) outside the {tiles.kinds} of the buffer")
    for k in range(nkinds):
        x = bf16_tiles(tiles, kind0 + k)
        is_v = v_period > 0 and k % v_period == v_slot
        dst.codes[kind0 + k], dst.scales[kind0 + k] = convert_v(x) if is_v else convert_qk(x)
    _count("head_tiles_fp8", (nkinds, tiles.heads, dst.tiles_per_head))
    return dst


def v_in_key_order(codes: torch.Tensor) -> torch.Tensor:
    """[.., 128 channels, 128 positions] -> [.., 128 keys, 128 channels]."""
    out = torch.empty_like(codes.transpose(-1, -2))
    out[..., vt8_key(torch.arange(128, device=codes.device)), :] = codes.transpose(-1, -2)
    return out


def attn_tiles_fp8(q, kv, out, *, q_kind=0, k_kind=1, v_kind=2, Lk, num_seqs, kv_lens=None, softmax_scale=None,
                   out_scatter=None, out_ld=None, out_map=None):
    if not isinstance(q, HeadTilesFp8) or not isinstance(kv, HeadTilesFp8):
        raise OsbError("attn_tiles_fp8: q and kv must be HeadTilesFp8 buffers")
    _need(out, torch.bfloat16, "out"); _need(kv_lens, torch.int32, "kv_lens")
    assert out_scatter is None, "the CPU double writes local outputs only"
    m, km = q.map, kv.map
    if kv_lens is not None and m.G > 1:
        raise OsbError("attn_tiles_fp8: kv_lens applies to unpacked query maps only (G == 1); packed sequences see all Lk keys")
    if out_map is not None:
        assert out_map.key()[4:] == m.key()[4:] and out_map.L == m.L
    om = out_map if out_map is not None else m
    H, D, dev = q.heads, q.head_dim, out.device
    sc = (softmax_scale if softmax_scale is not None else D ** -0.5) * 1.4426950408889634
    nsets = -(-num_seqs // m.G) if m.G > 1 else num_seqs
    nq = nsets * m.tps
    BK, nkb = km.tile_rows, km.tps
    qt = torch.arange(nq, device=dev)
    sets, qpos = qt // m.tps, qt % m.tps
    keys = torch.full((nsets,), m.G * Lk if m.G > 1 else Lk, dtype=torch.long, device=dev)
    if kv_lens is not None:
        keys = torch.minimum(keys, kv_lens.to(dev).long().clamp(min=0))
    # query rows of every tile: sequence, position, validity, key range [lo, hi)
    r = torch.arange(128, device=dev)[None]
    if m.G > 1:
        g = r // m.L
        seq, pos = sets[:, None] * m.G + g, (r % m.L).expand(nq, 128)
        valid = (g < m.G) & (seq < num_seqs)
        lo, hi = g * Lk, g * Lk + Lk
    else:
        seq, pos = sets[:, None].expand(nq, 128), qpos[:, None] * m.tile_rows + r
        valid = (r < m.tile_rows) & (pos < m.L)
        lo, hi = torch.zeros_like(pos), keys[sets][:, None].expand(nq, 128)
    lo, hi = torch.where(valid, lo, 0), torch.where(valid, hi, 0)
    qd = q.codes[q_kind, :, :nq].float()                                  # [H, nq, 128, 128]
    sq = q.scales[q_kind, :, :nq] * sc                                    # [H, nq, 128]
    mrun = torch.full((H, nq, 128, 1), float("-inf"), device=dev)
    l = torch.zeros(H, nq, 128, 1, device=dev)
    o = torch.zeros(H, nq, 128, 128, device=dev)
    nkt = (keys + BK - 1) // BK
    for kb in range(nkb):
        ti = sets * nkb + kb
        kd = kv.codes[k_kind, :, ti].float()                              # [H, nq, 128, 128]
        vd = v_in_key_order(kv.codes[v_kind, :, ti]).float()
        s = (qd @ kd.transpose(-1, -2)) * sq[..., None] * kv.scales[k_kind, :, ti][:, :, None, :]
        slot = kb * BK + torch.arange(128, device=dev)
        ok = ((slot[None, None] < kb * BK + BK) & (slot[None, None] >= lo[..., None]) & (slot[None, None] < hi[..., None])
              & (kb < nkt[sets])[:, None, None])
        s = s.masked_fill(~ok[None], float("-inf"))
        mn = torch.maximum(mrun, s.amax(-1, keepdim=True))
        fin = mn != float("-inf")
        alpha = torch.where(fin, torch.exp2(mrun - torch.where(fin, mn, 0)), torch.ones_like(mn))
        p = torch.exp2(s - torch.where(fin, mn, 0))
        l = l * alpha + p.sum(-1, keepdim=True)
        part = _e4m3(256.0 * p).float() @ vd
        o = o * alpha + kv.scales[v_kind, :, ti][:, :, None, :] * part
        mrun = mn
    res = torch.where(l > 0, o / (256.0 * l), torch.zeros_like(o))[..., :D]   # [H, nq, 128, D]
    seq_v, pos_v = seq[valid], pos[valid]   # -> rows of `out`: tiles.cuh row_of_token under the output map
    orow = seq_v * om.L + pos_v if om.mode == 0 else ((seq_v // om.S) * om.T + pos_v) * om.S + seq_v % om.S
    out[orow] = res.permute(1, 2, 0, 3)[valid].reshape(-1, H * D).to(torch.bfloat16)
    _count("attn_tiles_fp8", (num_seqs, m.L, Lk, H, D))
    return out


# ---- causal 3D VAE ops (NDHWC) ---------------------------------------------------------------------------------
def group_stats(x, groups: int, eps: float = 1e-6):
    _need(x, torch.bfloat16, "x")
    assert x.dim() == 5 and x.is_contiguous()
    nb, C = x.shape[0], x.shape[-1]
    if groups <= 0 or C % groups or C % 8 or 256 % (C // 8) or groups > 1024:
        raise OsbError(f"osb_group_stats failed (-1): C/8 must divide 256 and groups C (C = {C}, groups {groups})")
    xf = x.float().reshape(nb, -1, groups, C // groups)
    mean = xf.mean(dim=(1, 3))
    var = (xf - mean[:, None, :, None]).pow(2).mean(dim=(1, 3))
    _count("group_stats", tuple(x.shape), launches=2)   # block partials + fp64 finalize
    return torch.stack((mean, torch.rsqrt(var + eps)), dim=-1)


def vae_prep(x, *, stats=None, gamma=None, beta=None, groups: int = 32, silu: bool = False, up=(1, 1, 1), pad=(0, 0, 0),
             cp=None, slack_bytes: int = 128):
    _need(x, torch.bfloat16, "x"); _need(stats, torch.float32, "stats"); _need(gamma, torch.bfloat16, "gamma")
    _need(beta, torch.bfloat16, "beta")
    assert x.dim() == 5 and x.is_contiguous()
    nb, T, H, W, C = x.shape
    cp = cp or C
    if C % 8 or cp % 8 or cp < C:
        raise OsbError(f"osb_vae_prep failed (-1): channels must be multiples of 8 (c {C} cp {cp})")
    if any(f not in (1, 2) for f in up):
        raise OsbError(f"osb_vae_prep failed (-1): upsample factors must be 1 or 2, got {tuple(up)}")
    if stats is not None and (gamma is None or beta is None or groups <= 0 or C % groups):
        raise OsbError("osb_vae_prep failed (-1): GroupNorm needs gamma, beta and a valid group count")
    y = x.float()
    if stats is not None:
        cg = C // groups
        mean = stats[..., 0].repeat_interleave(cg, dim=1)[:, None, None, None, :]
        rstd = stats[..., 1].repeat_interleave(cg, dim=1)[:, None, None, None, :]
        y = (y - mean) * rstd * gamma.float() + beta.float()
    if silu:
        y = y * torch.sigmoid(y)
    ft, fh, fw = up
    if ft > 1:   # first-frame rule: frame 0 once, every later frame ft times (T' = 1 + ft (T - 1))
        y = torch.cat((y[:, :1], y[:, 1:].repeat_interleave(ft, dim=1)), dim=1)
    if fh > 1:
        y = y.repeat_interleave(fh, dim=2)
    if fw > 1:
        y = y.repeat_interleave(fw, dim=3)
    pt, ph, pw = pad
    if pt or ph or pw:   # replicate: T at the front only (causal), H / W on both sides
        y = F.pad(y.permute(0, 4, 1, 2, 3), (pw, pw, ph, ph, pt, 0), mode="replicate").permute(0, 2, 3, 4, 1)
    if cp > C:
        y = F.pad(y, (0, cp - C))
    _count("vae_prep", (tuple(x.shape), up, pad))
    return y.to(torch.bfloat16).contiguous()


def conv3d(x_pad, w_packed, bias, *, out_thw, stride=(1, 1, 1), taps=(3, 3, 3), narrow: bool = False, residual=None,
           block_n: int = 0):
    for t, n in ((x_pad, "x_pad"), (w_packed, "w_packed"), (bias, "bias"), (residual, "residual")):
        _need(t, torch.bfloat16, n)
    nb, tp, hp, wp, cp = x_pad.shape
    kt, kh, kw = taps
    cout = w_packed.shape[0]
    if any(s not in (1, 2) for s in stride):
        raise OsbError(f"osb_conv3d_ndhwc failed (-1): strides must be 1 or 2, got {tuple(stride)}")
    if any(k not in (1, 2, 3) for k in taps):
        raise OsbError(f"osb_conv3d_ndhwc failed (-1): taps must be 1..3, got {tuple(taps)}")
    if cout % 8:
        raise OsbError(f"osb_conv3d_ndhwc: Cout must be a multiple of 8 (pad the weights), got {cout}")
    if narrow:
        if cp not in (8, 16) or kw * cp > 64:
            raise OsbError("osb_conv3d_ndhwc: narrow mode needs Cp in {8,16} with kw*Cp <= 64")
        w = w_packed.float().view(cout, kt * kh, 64)[:, :, : kw * cp].reshape(cout, kt, kh, kw, cp)
    else:
        if cp % 64:
            raise OsbError(f"osb_conv3d_ndhwc: Cp must be a multiple of 64 (or use narrow mode), got {cp}")
        w = w_packed.float().view(cout, kt, kh, kw, cp)
    t_out, h_out, w_out = out_thw
    st, sh, sw = stride
    if (t_out - 1) * st + kt > tp or (h_out - 1) * sh + kh > hp or (w_out - 1) * sw + kw > wp:
        raise OsbError("osb_conv3d_ndhwc: padded input too small for the output")
    y = F.conv3d(x_pad.to(ACC_DTYPE).permute(0, 4, 1, 2, 3), w.to(ACC_DTYPE).permute(0, 4, 1, 2, 3), None, stride=stride)
    y = y[:, :, :t_out, :h_out, :w_out].permute(0, 2, 3, 4, 1)
    if bias is not None:
        y = y + bias.to(ACC_DTYPE)
    if residual is not None:
        y = y + residual.to(ACC_DTYPE)
    _count("conv3d", (tuple(x_pad.shape), cout, stride, narrow))
    return y.to(torch.bfloat16).contiguous()


def pack_conv_weight(w, cp: int, narrow: bool, cout_pad=None):
    cout, cin, kt, kh, kw = w.shape
    co = cout_pad or cout
    if narrow:
        out = torch.zeros(co, kt * kh, 64, dtype=w.dtype, device=w.device)
        blk = torch.zeros(cout, kt * kh, kw, cp, dtype=w.dtype, device=w.device)
        blk[..., :cin] = w.permute(0, 2, 3, 4, 1).reshape(cout, kt * kh, kw, cin)
        out[:cout, :, : kw * cp] = blk.reshape(cout, kt * kh, kw * cp)
        return out.reshape(co, kt * kh * 64).to(torch.bfloat16).contiguous()
    out = torch.zeros(co, kt, kh, kw, cp, dtype=w.dtype, device=w.device)
    out[:cout, ..., :cin] = w.permute(0, 2, 3, 4, 1)
    return out.reshape(co, kt * kh * kw * cp).to(torch.bfloat16).contiguous()


def cfg_euler(cond, uncond, uncond2, x, *, g_txt: float, g_img: float = 1.0, g_img_map=None, dt: float, out=None):
    for t, n in ((cond, "cond"), (uncond, "uncond"), (uncond2, "uncond2"), (x, "x"), (g_img_map, "g_img_map")):
        _need(t, torch.bfloat16, n)
    if x.numel() % 8 or (g_img_map is not None and (g_img_map.numel() % 8 or x.numel() % g_img_map.numel())):
        raise OsbError("osb_cfg_euler failed (-1): element count and guidance map period must be multiples of 8, "
                       "the period dividing the count")
    c, u = cond.float(), uncond.float()
    if uncond2 is None:
        pred = u + g_txt * (c - u)
    else:
        u2 = uncond2.float()
        gi = g_img if g_img_map is None else g_img_map.float().reshape(-1).repeat(x.numel() // g_img_map.numel()).view_as(x)
        pred = u2 + gi * (u - u2) + g_txt * (c - u)
    y = (x.float() + dt * pred).to(torch.bfloat16)
    _count("cfg_euler", x.numel())
    return _put(y, out)


def rf_masked_step(vc, vu, z, frame_mask, t_cur, t_next, *, guidance: float, noise=None, update: bool = True,
                   num_timesteps: int = 1000, out=None):
    """osb_rf_masked_step with the kernel's rounding points: fp32 math, one rounding to bf16, frames left alone copied
    exactly."""
    for t, n in ((vc, "vc"), (vu, "vu"), (z, "z"), (noise, "noise"), (out, "out")):
        _need(t, torch.bfloat16, n)
        if t is not None and t.shape != z.shape:
            raise OsbError(f"{n} must have the latent's shape")
    for t, n in ((frame_mask, "frame_mask"), (t_cur, "t_cur"), (t_next, "t_next")):
        _need(t, torch.float32, n)
    if update and (vc is None or vu is None):
        raise OsbError("osb_rf_masked_step failed (-1): the update needs cond and uncond")
    if not update and noise is None:
        raise OsbError("osb_rf_masked_step failed (-1): without the update there must be noise to add")
    N = float(num_timesteps)   # dt and t/N multiply by fl(1/N), as the kernel (and torch's scalar division on CUDA) do
    per_frame = lambda f: f[:, None, :, None, None]  # noqa: E731  [B, T] -> broadcast over [B, C, T, H, W]
    per_sample = lambda v: v[:, None, None, None, None]  # noqa: E731
    m = frame_mask * N
    x = z.float()
    if update:
        upd = m >= t_cur[:, None]
        c, u = vc.float(), vu.float()
        x = torch.where(per_frame(upd), x + per_sample((t_cur - t_next) * (1.0 / N)) * (u + guidance * (c - u)), x)
        prev = upd
    else:
        prev = frame_mask == 1
    if noise is not None:
        add = (m >= t_next[:, None]) & ~prev
        a = per_sample(t_next * (1.0 / N))
        x = torch.where(per_frame(add), (1.0 - a) * x + a * noise.float(), x)
    y = x.to(torch.bfloat16)   # frames left alone round-trip bf16 -> fp32 -> bf16 exactly
    _count("rf_masked_step", (tuple(z.shape), bool(update), noise is not None))
    return _put(y, out)
