"""ctypes binding of libosb200.so (the C ABI in include/osb200.h).

PyTorch is used only for device memory and streams: every op takes torch CUDA tensors, passes
raw device pointers + the current stream to the library and returns the output tensor.  There is
NO fallback: importing without the built library, or calling an op on a non-CUDA tensor, raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OSB200_LIB", os.path.join(_HERE, "libosb200.so"))  # override: another build of the library

# every symbol include/osb200.h declares (tests check the library exports all of them)
EXPORTS = (
    "osb_init",
    "osb_version",
    "osb_last_error",
    "osb_launch_count",
    "osb_ln_modulate",
    "osb_gemm_bf16",
    "osb_attn_short",
    "osb_conv3d_ndhwc",
    "osb_group_stats",
    "osb_group_stats_workspace_bytes",
    "osb_vae_prep",
    "osb_cfg_euler",
    "osb_gemm_head_tiles",
    "osb_head_tiles_per_head",
    "osb_attn_tiles",
    "osb_tmap_cache_stats",
    "osb_ln_modulate_scatter",
    "osb_comm_barrier",
    "osb_rf_masked_step",
    "osb_gemm_lora",
    "osb_attn_short_bias",
    "osb_rms_norm",
    "osb_gemm_fp8",
    "osb_ln_modulate_fp8",
    "osb_quant_rows_fp8",
    "osb_gemm_fp8_blocks",
    "osb_quant_blocks_fp8",
    "osb_attn_fp8",
    "osb_head_tiles_fp8",
    "osb_attn_tiles_fp8",
    "osb_attn_frames",
)

EPI_BIAS, EPI_BIAS_GELU_TANH, EPI_BIAS_GATE_RES = 0, 1, 2
EPI_GATED_GELU, EPI_BIAS_QUICK_GELU = 3, 4
EPI_BIAS_GELU_TANH_FP8 = 5   # gemm_fp8_blocks only: GELU-tanh emitted as e4m3 codes with 1 x 128 block scales


class OsbError(RuntimeError):
    pass


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise OsbError(
            f"{LIB_PATH} is missing: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "osb200 has no CPU or PyTorch fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise OsbError(f"libosb200.so does not export {name}")
    lib.osb_last_error.restype = C.c_char_p
    lib.osb_launch_count.restype = C.c_int64
    lib.osb_init.argtypes = [C.c_int]
    lib.osb_ln_modulate.argtypes = [
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p,
        C.c_int64, C.c_float, C.c_void_p,
    ]
    lib.osb_gemm_bf16.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_gemm_lora.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.osb_gemm_fp8.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_ln_modulate_fp8.argtypes = [
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p,
        C.c_int64, C.c_float, C.c_void_p,
    ]
    lib.osb_quant_rows_fp8.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int,
                                       C.c_void_p]
    lib.osb_gemm_fp8_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.osb_quant_blocks_fp8.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64,
                                         C.c_int, C.c_int, C.c_void_p]
    lib.osb_attn_short.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_attn_short_bias.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.osb_attn_fp8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.osb_attn_frames.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_rms_norm.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_void_p]
    lib.osb_conv3d_ndhwc.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_vae_prep.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_cfg_euler.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float,
                                  C.c_float, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]
    lib.osb_group_stats.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                    C.c_int64, C.c_void_p, C.c_void_p]
    lib.osb_group_stats_workspace_bytes.argtypes = [C.c_int64, C.c_int64, C.c_int32]
    lib.osb_group_stats_workspace_bytes.restype = C.c_int64
    lib.osb_gemm_head_tiles.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.osb_attn_tiles.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_head_tiles_fp8.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_attn_tiles_fp8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.osb_head_tiles_per_head.argtypes = [C.c_void_p, C.c_int64]
    lib.osb_head_tiles_per_head.restype = C.c_int64
    lib.osb_tmap_cache_stats.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_tmap_cache_stats.restype = None
    lib.osb_ln_modulate_scatter.argtypes = [
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_float,
        C.c_void_p, C.c_void_p,
    ]
    lib.osb_comm_barrier.argtypes = [C.c_void_p, C.c_void_p]
    lib.osb_rf_masked_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_float, C.c_int32,
                                       C.c_int32, C.c_void_p]
    return lib


_lib = _load()
_initialised_devices: set[int] = set()

# Optional per-launch device timing (bench.py's roofline leg): when a list is installed with
# start_profile(), every op brackets its launch with CUDA events on the launching stream and appends
# (kernel family, algorithmic work, start_event, end_event).  Off (None) in normal operation.
_profile: list | None = None


def start_profile() -> None:
    global _profile
    _profile = []


def stop_profile() -> list:
    """Returns [(family, work, milliseconds)] after synchronising."""
    global _profile
    import torch

    torch.cuda.synchronize()
    rec, _profile = _profile or [], None
    return [(n, w, s.elapsed_time(e)) for (n, w, s, e) in rec]


class _Timed:
    def __init__(self, family: str, work: float):
        self.family, self.work = family, work

    def __enter__(self):
        if _profile is not None:
            import torch

            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
        return self

    def __exit__(self, *exc):
        if _profile is not None:
            self.e.record()
            _profile.append((self.family, self.work, self.s, self.e))
        return False


class GemmArgs(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("W", C.c_void_p), ("bias", C.c_void_p), ("D", C.c_void_p),
        ("R", C.c_void_p), ("gate", C.c_void_p), ("mod_index", C.c_void_p),
        ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
        ("lda", C.c_int64), ("ldw", C.c_int64), ("ldd", C.c_int64), ("ldr", C.c_int64),
        ("group_rows", C.c_int64), ("gate_stride", C.c_int64),
        ("epilogue", C.c_int32), ("cta_group", C.c_int32), ("block_n", C.c_int32), ("reserved", C.c_int32),
    ]


class LoraArgs(C.Structure):
    _fields_ = [("U", C.c_void_p), ("B", C.c_void_p), ("ldu", C.c_int64), ("ldb", C.c_int64), ("r", C.c_int32),
                ("reserved", C.c_int32), ("col_scale", C.c_void_p)]


class GemmFp8Args(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("W", C.c_void_p), ("a_scale", C.c_void_p), ("w_scale", C.c_void_p),
        ("bias", C.c_void_p), ("D", C.c_void_p), ("R", C.c_void_p), ("gate", C.c_void_p), ("mod_index", C.c_void_p),
        ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
        ("lda", C.c_int64), ("ldw", C.c_int64), ("ldd", C.c_int64), ("ldr", C.c_int64),
        ("group_rows", C.c_int64), ("gate_stride", C.c_int64),
        ("epilogue", C.c_int32), ("block_n", C.c_int32),
    ]


class Fp8BlocksArgs(C.Structure):
    _fields_ = [("a_scale_ld", C.c_int64), ("D8", C.c_void_p), ("d_scale", C.c_void_p), ("ldd8", C.c_int64),
                ("ld_dscale", C.c_int64)]


class AttnShortArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("q_ld", C.c_int64), ("k_ld", C.c_int64), ("v_ld", C.c_int64), ("out_ld", C.c_int64),
        ("num_seqs", C.c_int64), ("seqs_per_batch", C.c_int64),
        ("q_batch_stride", C.c_int64), ("q_seq_stride", C.c_int64), ("q_tok_stride", C.c_int64),
        ("k_batch_stride", C.c_int64), ("k_seq_stride", C.c_int64), ("k_tok_stride", C.c_int64),
        ("Lq", C.c_int32), ("Lk", C.c_int32),
        ("kv_lens", C.c_void_p),
        ("num_heads", C.c_int32), ("head_dim", C.c_int32),
        ("q_norm_w", C.c_void_p), ("k_norm_w", C.c_void_p),
        ("norm_eps", C.c_float),
        ("rope_cos", C.c_void_p), ("rope_sin", C.c_void_p),
        ("softmax_scale", C.c_float),
        ("q_norm_w2", C.c_void_p), ("k_norm_w2", C.c_void_p), ("norm_split", C.c_int32), ("reserved", C.c_int32),
        ("rope_half", C.c_int32), ("reserved2", C.c_int32),
    ]


class AttnFramesArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("q_ld", C.c_int64), ("k_ld", C.c_int64), ("v_ld", C.c_int64), ("out_ld", C.c_int64),
        ("q_batch_stride", C.c_int64), ("k_batch_stride", C.c_int64),
        ("Lq", C.c_int64), ("Lk", C.c_int64),
        ("batch", C.c_int32), ("head_dim", C.c_int32), ("frame_tokens", C.c_int32), ("q_frame0", C.c_int32),
        ("softmax_scale", C.c_float), ("reserved", C.c_int32),
    ]


class Conv3dArgs(C.Structure):
    _fields_ = [
        ("x_pad", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("y", C.c_void_p), ("residual", C.c_void_p),
        ("nb", C.c_int32), ("tp", C.c_int32), ("hp", C.c_int32), ("wp", C.c_int32), ("cp", C.c_int32),
        ("t_out", C.c_int32), ("h_out", C.c_int32), ("w_out", C.c_int32), ("cout", C.c_int32),
        ("st", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("narrow", C.c_int32), ("block_n", C.c_int32),
    ]


class VaePrepArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("y", C.c_void_p), ("mean_rstd", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("nb", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32),
        ("groups", C.c_int32), ("silu", C.c_int32),
        ("ft", C.c_int32), ("fh", C.c_int32), ("fw", C.c_int32),
        ("pad_t", C.c_int32), ("pad_h", C.c_int32), ("pad_w", C.c_int32),
        ("cp", C.c_int32),
    ]


def last_error() -> str:
    return _lib.osb_last_error().decode()


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise OsbError(f"{what} failed ({rc}): {last_error()}")


def version() -> int:
    return _lib.osb_version()


def launch_count() -> int:
    return int(_lib.osb_launch_count())


def init(device: int | None = None) -> None:
    import torch

    if not torch.cuda.is_available():
        raise OsbError("osb200 needs a CUDA device (sm_90a); there is no CPU path")
    if device is None:
        device = torch.cuda.current_device()
    if device in _initialised_devices:
        return
    torch.cuda.init()
    _check(_lib.osb_init(int(device)), "osb_init")
    _initialised_devices.add(device)


def _stream():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _need(t, dtype, name):
    import torch

    if t is None:
        return
    if not t.is_cuda:
        raise OsbError(f"{name} must be a CUDA tensor (osb200 has no CPU path)")
    if t.dtype != dtype:
        raise OsbError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() >= 1 and t.stride(-1) != 1 and t.shape[-1] != 1:
        raise OsbError(f"{name} must have unit stride in the last dimension")
    init(t.device.index)


def require_cuda_bf16(t, what: str) -> None:
    """The product path has no CPU / eager fallback: the host-side models call this on entry so that a model left on the
    CPU or in another dtype fails loudly instead of silently running somewhere else."""
    import torch

    if not t.is_cuda or t.dtype != torch.bfloat16:
        raise OsbError(f"{what} (osb200) runs on CUDA in bfloat16 only: call .cuda().to(torch.bfloat16); "
                       "there is no CPU / eager fallback")


MAX_PEERS = 16


class Scatter(C.Structure):
    """include/osb200.h `osb_scatter`: output rows viewed as [B, I, J] are routed to peer buffers (sequence parallel)."""
    _fields_ = [("mode", C.c_int32), ("P", C.c_int32), ("rank", C.c_int32), ("I", C.c_int32), ("J", C.c_int32),
                ("reserved", C.c_int32 * 3), ("peer", C.c_void_p * MAX_PEERS)]


class CommBarrierArgs(C.Structure):
    _fields_ = [("P", C.c_int32), ("rank", C.c_int32), ("epoch", C.c_void_p), ("flags_local", C.c_void_p),
                ("flags_peer", C.c_void_p * MAX_PEERS)]


def make_scatter(mode: int, P: int, rank: int, I: int, J: int, peer_ptrs) -> Scatter:
    sc = Scatter()
    sc.mode, sc.P, sc.rank, sc.I, sc.J = mode, P, rank, I, J
    for i, ptr in enumerate(peer_ptrs):   # raw (peer-mapped) device pointers, or local tensors
        sc.peer[i] = int(ptr) if isinstance(ptr, int) else ptr.data_ptr()
    return sc


def comm_barrier(P: int, rank: int, epoch, flags_local_ptr: int, flags_peer_ptrs) -> None:
    """Cross-rank ordering point of a peer-memory exchange (osb_comm_barrier): enqueued on the current stream."""
    import torch

    _need(epoch, torch.int32, "epoch")
    a = CommBarrierArgs()
    a.P, a.rank, a.epoch, a.flags_local = P, rank, epoch.data_ptr(), int(flags_local_ptr)
    for i, ptr in enumerate(flags_peer_ptrs):
        a.flags_peer[i] = int(ptr)
    _check(_lib.osb_comm_barrier(C.byref(a), _stream()), "osb_comm_barrier")


def ln_modulate(x, shift, scale, *, group_rows: int, mod_index=None, eps: float = 1e-6, out=None, scatter: Scatter | None = None):
    """y = LN(x) * (1 + scale[g]) + shift[g];  x bf16 [rows, C]; shift/scale fp32 [G, C] views.  With `scatter` the rows
    are stored straight into peer buffers (osb_ln_modulate_scatter) and nothing is returned."""
    import torch

    _need(x, torch.bfloat16, "x"); _need(shift, torch.float32, "shift"); _need(scale, torch.float32, "scale")
    _need(mod_index, torch.int32, "mod_index")
    assert x.dim() == 2 and x.is_contiguous()
    assert shift.dim() == 2 and scale.dim() == 2 and shift.stride(0) == scale.stride(0)
    rows, Cdim = x.shape
    if scatter is not None:
        with _Timed("ln_modulate", 4.0 * rows * Cdim):
            _check(_lib.osb_ln_modulate_scatter(_ptr(x), _ptr(shift), _ptr(scale), rows, Cdim, group_rows, _ptr(mod_index),
                                                shift.stride(0), eps, C.byref(scatter), _stream()), "osb_ln_modulate_scatter")
        return None
    if out is None:
        out = torch.empty_like(x)
    with _Timed("ln_modulate", 4.0 * rows * Cdim):  # algorithmic bytes: read x + write y (bf16)
        _check(_lib.osb_ln_modulate(_ptr(x), _ptr(shift), _ptr(scale), _ptr(out), rows, Cdim, group_rows,
                                    _ptr(mod_index), shift.stride(0), eps, _stream()), "osb_ln_modulate")
    return out


def rms_norm(x, w, *, eps: float = 1e-6, out=None):
    """y = bf16(w * bf16(x * rsqrt(mean(x^2) + eps))) per row (osb_rms_norm, T5LayerNorm); x bf16 [rows, C], w bf16 [C]."""
    import torch

    _need(x, torch.bfloat16, "x"); _need(w, torch.bfloat16, "w")
    if x.dim() != 2 or not x.is_contiguous() or w.shape != (x.shape[1],):
        raise OsbError(f"rms_norm: x must be a contiguous [rows, C] tensor and w [C], got {tuple(x.shape)} and {tuple(w.shape)}")
    if out is None:
        out = torch.empty_like(x)
    rows, Cdim = x.shape
    with _Timed("rms_norm", 4.0 * rows * Cdim):  # algorithmic bytes: read x + write y (bf16)
        _check(_lib.osb_rms_norm(_ptr(x), _ptr(w), _ptr(out), rows, Cdim, eps, _stream()), "osb_rms_norm")
    return out


def _epilogue_shapes(fn, M, N, out_cols, out, bias, residual, gate, group_rows, mod_index):
    """Extents of the optional GEMM operands.  The kernels address out, bias, residual, gate and mod_index by (row,
    column) with only a row stride, so a tensor smaller than the problem would be read or written out of bounds: refuse
    it here.  mod_index's values live on the device and are not checked."""
    if out is not None and tuple(out.shape) != (M, out_cols):
        raise OsbError(f"{fn}: out must be [{M}, {out_cols}], got {tuple(out.shape)}")
    if bias is not None and tuple(bias.shape) != (N,):
        raise OsbError(f"{fn}: bias must be [{N}], got {tuple(bias.shape)}")
    if residual is not None and tuple(residual.shape) != (M, N):
        raise OsbError(f"{fn}: residual must be [{M}, {N}], got {tuple(residual.shape)}")
    groups = -(-M // (group_rows if group_rows > 0 else M))
    if gate is not None and (gate.dim() != 2 or gate.shape[1] != N or (mod_index is None and gate.shape[0] < groups)):
        raise OsbError(f"{fn}: gate must be [G, {N}] with G >= {groups} row groups (or indexed by mod_index), got "
                       f"{tuple(gate.shape)}")
    if mod_index is not None and (mod_index.dim() != 1 or mod_index.shape[0] < groups):
        raise OsbError(f"{fn}: mod_index must be 1-D with at least {groups} entries, got {tuple(mod_index.shape)}")


def _gemm_args(a, w, bias, epilogue, residual, gate, group_rows, mod_index, out, cta_group, block_n, fn="gemm"):
    import torch

    _need(a, torch.bfloat16, "a"); _need(w, torch.bfloat16, "w"); _need(bias, torch.bfloat16, "bias")
    _need(residual, torch.bfloat16, "residual"); _need(gate, torch.float32, "gate")
    _need(mod_index, torch.int32, "mod_index")
    if a.dim() != 2 or w.dim() != 2 or a.shape[1] != w.shape[1]:
        raise OsbError(f"{fn}: a [M, K] and w [N, K] expected, got {tuple(a.shape)} and {tuple(w.shape)}")
    M, K = a.shape
    N = w.shape[0]
    _epilogue_shapes(fn, M, N, N // 2 if epilogue == EPI_GATED_GELU else N, out, bias, residual, gate, group_rows,
                     mod_index)
    if out is None:   # the gated GELU writes one column per (wi_0, wi_1) row pair of w
        out = torch.empty((M, N // 2 if epilogue == EPI_GATED_GELU else N), dtype=torch.bfloat16, device=a.device)
    _need(out, torch.bfloat16, "out")
    args = GemmArgs()
    args.A, args.W, args.bias, args.D = a.data_ptr(), w.data_ptr(), (bias.data_ptr() if bias is not None else None), out.data_ptr()
    args.R = residual.data_ptr() if residual is not None else None
    args.gate = gate.data_ptr() if gate is not None else None
    args.mod_index = mod_index.data_ptr() if mod_index is not None else None
    args.M, args.N, args.K = M, N, K
    args.lda, args.ldw, args.ldd = a.stride(0), w.stride(0), out.stride(0)
    args.ldr = residual.stride(0) if residual is not None else 0
    args.group_rows = group_rows if group_rows > 0 else M
    args.gate_stride = gate.stride(0) if gate is not None else 0
    args.epilogue, args.cta_group, args.block_n = epilogue, cta_group, block_n
    return args, out


def gemm(a, w, bias=None, *, epilogue: int = EPI_BIAS, residual=None, gate=None, group_rows: int = 0,
         mod_index=None, out=None, cta_group: int = 0, block_n: int = 0):
    """out = epilogue(a @ w.T + bias).  a bf16 [M,K] (row stride free), w bf16 [N,K], bias bf16 [N].
    GATE_RES: out = residual + gate[g] * (a @ w.T + bias), gate fp32 [G, N] view, may be None.
    GATED_GELU: out [M, N/2], out[:, c] = gelu_tanh(p[:, 2c]) * p[:, 2c+1], p = a @ w.T + bias (w's rows interleave
    T5's wi_0 and wi_1, see interleave_gated).  BIAS_QUICK_GELU: out = p * sigmoid(1.702 p) (CLIP)."""
    args, out = _gemm_args(a, w, bias, epilogue, residual, gate, group_rows, mod_index, out, cta_group, block_n)
    with _Timed("gemm", 2.0 * args.M * args.N * args.K):  # algorithmic FLOPs
        _check(_lib.osb_gemm_bf16(C.byref(args), _stream()), "osb_gemm_bf16")
    return out


def gemm_lora(a, w, bias, u, b, *, epilogue: int = EPI_BIAS, residual=None, gate=None, group_rows: int = 0,
              mod_index=None, out=None, block_n: int = 0, col_scale=None):
    """out = epilogue(a @ w.T + u @ b.T + bias) in one fp32 accumulator (osb_gemm_lora): `gemm` plus an unmerged LoRA
    update.  u bf16 [M, r] = x @ lora_A.T (the down projection, row stride free), b bf16 [N, r] = scaling * lora_B; r is
    a multiple of 8 (zero-pad A's rows and B's columns).  col_scale: None, or a contiguous fp32 [N] tensor g on a's
    device: out = epilogue(g * (a @ w.T + u @ b.T) + bias), DoRA's per-output-channel factor."""
    import torch

    _need(u, torch.bfloat16, "u"); _need(b, torch.bfloat16, "b")
    if u.dim() != 2 or b.dim() != 2 or u.shape[0] != a.shape[0] or b.shape[0] != w.shape[0] or u.shape[1] != b.shape[1]:
        raise OsbError(f"gemm_lora: u must be [M, r] and b [N, r] for a {tuple(a.shape)} x {tuple(w.shape)} GEMM, got "
                       f"{tuple(u.shape)} and {tuple(b.shape)}")
    if col_scale is not None:
        if col_scale.dtype != torch.float32 or col_scale.shape != (w.shape[0],) or not col_scale.is_contiguous() \
                or col_scale.device != a.device:
            raise OsbError(f"gemm_lora: col_scale must be a contiguous float32 [{w.shape[0]}] tensor on {a.device}, got "
                           f"{col_scale.dtype} {tuple(col_scale.shape)} on {col_scale.device}")
    args, out = _gemm_args(a, w, bias, epilogue, residual, gate, group_rows, mod_index, out, 0, block_n, "gemm_lora")
    la = LoraArgs()
    la.U, la.B, la.ldu, la.ldb, la.r = u.data_ptr(), b.data_ptr(), u.stride(0), b.stride(0), u.shape[1]
    la.col_scale = None if col_scale is None else col_scale.data_ptr()
    with _Timed("gemm", 2.0 * args.M * args.N * (args.K + la.r)):
        _check(_lib.osb_gemm_lora(C.byref(args), C.byref(la), _stream()), "osb_gemm_lora")
    return out


# ---- FP8 (e4m3) with per-row scales (include/osb200.h): s[r] = amax(|X[r, :]|) / 448 (1 for a zero row), codes
# e4m3_rn_satfinite(X / s).  e4m3 tensors are torch.float8_e4m3fn, scales fp32. ---------------------------------------
def gemm_fp8(a8, a_scale, w8, w_scale, bias=None, *, epilogue: int = EPI_BIAS, residual=None, gate=None,
             group_rows: int = 0, mod_index=None, out=None, block_n: int = 0):
    """out = epilogue(acc * (a_scale[m] * w_scale[n]) + bias), acc = a8 @ w8.T summed in fp32 (osb_gemm_fp8).
    a8 e4m3 [M, K] (row stride free), w8 e4m3 [N, K], scales fp32 [M] / [N]; K % 128 == 0.  The epilogues BIAS,
    BIAS_GELU_TANH and BIAS_GATE_RES behave as in `gemm`."""
    import torch

    _need(a8, torch.float8_e4m3fn, "a8"); _need(w8, torch.float8_e4m3fn, "w8")
    _need(a_scale, torch.float32, "a_scale"); _need(w_scale, torch.float32, "w_scale")
    _need(bias, torch.bfloat16, "bias"); _need(residual, torch.bfloat16, "residual"); _need(gate, torch.float32, "gate")
    _need(mod_index, torch.int32, "mod_index")
    if a8.dim() != 2 or w8.dim() != 2 or a8.shape[1] != w8.shape[1]:
        raise OsbError(f"gemm_fp8: a8 [M, K] and w8 [N, K] expected, got {tuple(a8.shape)} and {tuple(w8.shape)}")
    M, K = a8.shape
    N = w8.shape[0]
    if a_scale is None or w_scale is None or a_scale.shape != (M,) or w_scale.shape != (N,):
        raise OsbError(f"gemm_fp8: a_scale must be [{M}] and w_scale [{N}]")
    _epilogue_shapes("gemm_fp8", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=a8.device)
    _need(out, torch.bfloat16, "out")
    g = GemmFp8Args()
    g.A, g.W, g.a_scale, g.w_scale = a8.data_ptr(), w8.data_ptr(), a_scale.data_ptr(), w_scale.data_ptr()
    g.bias = bias.data_ptr() if bias is not None else None
    g.D = out.data_ptr()
    g.R = residual.data_ptr() if residual is not None else None
    g.gate = gate.data_ptr() if gate is not None else None
    g.mod_index = mod_index.data_ptr() if mod_index is not None else None
    g.M, g.N, g.K = M, N, K
    g.lda, g.ldw, g.ldd = a8.stride(0), w8.stride(0), out.stride(0)
    g.ldr = residual.stride(0) if residual is not None else 0
    g.group_rows = group_rows if group_rows > 0 else M
    g.gate_stride = gate.stride(0) if gate is not None else 0
    g.epilogue, g.block_n = epilogue, block_n
    with _Timed("gemm_fp8", 2.0 * M * N * K):
        _check(_lib.osb_gemm_fp8(C.byref(g), _stream()), "osb_gemm_fp8")
    return out


def ln_modulate_fp8(x, shift, scale, *, group_rows: int, mod_index=None, eps: float = 1e-6, out=None, out_scale=None):
    """`ln_modulate` with the fp32 result quantized per row (osb_ln_modulate_fp8): returns (e4m3 [rows, C], fp32 [rows])."""
    import torch

    _need(x, torch.bfloat16, "x"); _need(shift, torch.float32, "shift"); _need(scale, torch.float32, "scale")
    _need(mod_index, torch.int32, "mod_index")
    assert x.dim() == 2 and x.is_contiguous()
    assert shift.dim() == 2 and scale.dim() == 2 and shift.stride(0) == scale.stride(0)
    rows, Cdim = x.shape
    if out is None:
        out = torch.empty((rows, Cdim), dtype=torch.float8_e4m3fn, device=x.device)
    if out_scale is None:
        out_scale = torch.empty(rows, dtype=torch.float32, device=x.device)
    _need(out, torch.float8_e4m3fn, "out"); _need(out_scale, torch.float32, "out_scale")
    if out.shape != (rows, Cdim) or not out.is_contiguous() or out_scale.shape != (rows,):
        raise OsbError(f"ln_modulate_fp8: out must be a contiguous [{rows}, {Cdim}] e4m3 tensor and out_scale [{rows}]")
    with _Timed("ln_modulate", 3.0 * rows * Cdim):  # algorithmic bytes: read x (bf16) + write codes (e4m3)
        _check(_lib.osb_ln_modulate_fp8(_ptr(x), _ptr(shift), _ptr(scale), _ptr(out), _ptr(out_scale), rows, Cdim,
                                        group_rows, _ptr(mod_index), shift.stride(0), eps, _stream()),
               "osb_ln_modulate_fp8")
    return out, out_scale


def quant_rows_fp8(x, *, out=None, out_scale=None):
    """Per-row e4m3 quantization of bf16 x [rows, K] (row stride free) in one pass (osb_quant_rows_fp8): returns
    (e4m3 [rows, K], fp32 [rows])."""
    import torch

    _need(x, torch.bfloat16, "x")
    if x.dim() != 2:
        raise OsbError(f"quant_rows_fp8: x must be [rows, K], got {tuple(x.shape)}")
    rows, K = x.shape
    if out is None:
        out = torch.empty((rows, K), dtype=torch.float8_e4m3fn, device=x.device)
    if out_scale is None:
        out_scale = torch.empty(rows, dtype=torch.float32, device=x.device)
    _need(out, torch.float8_e4m3fn, "out"); _need(out_scale, torch.float32, "out_scale")
    if out.shape != (rows, K) or out_scale.shape != (rows,):
        raise OsbError(f"quant_rows_fp8: out must be [{rows}, {K}] and out_scale [{rows}]")
    with _Timed("quant_rows_fp8", 3.0 * rows * K):  # algorithmic bytes: read bf16 + write e4m3
        _check(_lib.osb_quant_rows_fp8(_ptr(x), x.stride(0), _ptr(out), out.stride(0), _ptr(out_scale), rows, K,
                                       _stream()), "osb_quant_rows_fp8")
    return out, out_scale


# ---- FP8 (e4m3) with 1 x 128 block scales (include/osb200.h): the block (r, b) = X[r, 128 b : 128 b + 128] gets
# s[r, b] = amax(|block|) / 448 (1 for a zero block), codes e4m3_rn_satfinite(X / s).  Scale tensors may be column views
# of wider buffers (row stride free, unit column stride). ---------------------------------------------------------------
def _scale_view(t, rows: int, cols: int, name: str):
    import torch

    _need(t, torch.float32, name)
    if t is None or t.dim() != 2 or t.shape != (rows, cols):
        raise OsbError(f"{name} must be a float32 [{rows}, {cols}] tensor (row stride free), got "
                       f"{None if t is None else tuple(t.shape)}")
    return t.stride(0)


def gemm_fp8_blocks(a8, a_scale, w8, w_scale, bias=None, *, epilogue: int = EPI_BIAS, residual=None, gate=None,
                    group_rows: int = 0, mod_index=None, out=None, out_scale=None, block_n: int = 0):
    """`gemm_fp8` with block-scaled A (osb_gemm_fp8_blocks).  a_scale: fp32 [M] (per row: with a bf16 epilogue this is
    exactly `gemm_fp8`) or [M, K / 128] (block mode, row stride free): out = epilogue(w_scale[n] * sum_kb a_scale[m, kb]
    * acc_kb + bias).  EPI_BIAS, EPI_BIAS_GELU_TANH and EPI_BIAS_GATE_RES write bf16 `out` as in `gemm`.
    EPI_BIAS_GELU_TANH_FP8 writes e4m3 `out` [M, N] and fp32 `out_scale` [M, N / 128] (both row stride free, e.g. column
    slices of a wider buffer) and returns (out, out_scale); N % 128 == 0."""
    import torch

    _need(a8, torch.float8_e4m3fn, "a8"); _need(w8, torch.float8_e4m3fn, "w8"); _need(w_scale, torch.float32, "w_scale")
    _need(bias, torch.bfloat16, "bias"); _need(residual, torch.bfloat16, "residual"); _need(gate, torch.float32, "gate")
    _need(mod_index, torch.int32, "mod_index")
    if a8.dim() != 2 or w8.dim() != 2 or a8.shape[1] != w8.shape[1]:
        raise OsbError(f"gemm_fp8_blocks: a8 [M, K] and w8 [N, K] expected, got {tuple(a8.shape)} and {tuple(w8.shape)}")
    M, K = a8.shape
    N = w8.shape[0]
    if w_scale is None or w_scale.shape != (N,):
        raise OsbError(f"gemm_fp8_blocks: w_scale must be [{N}]")
    b = Fp8BlocksArgs()
    if a_scale is not None and a_scale.dim() == 1:
        _need(a_scale, torch.float32, "a_scale")
        if a_scale.shape != (M,):
            raise OsbError(f"gemm_fp8_blocks: a per-row a_scale must be [{M}], got {tuple(a_scale.shape)}")
    else:
        b.a_scale_ld = _scale_view(a_scale, M, K // 128, "a_scale")
    fp8_out = epilogue == EPI_BIAS_GELU_TANH_FP8
    _epilogue_shapes("gemm_fp8_blocks", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    if fp8_out:
        if out is None:
            out = torch.empty((M, N), dtype=torch.float8_e4m3fn, device=a8.device)
        if out_scale is None:
            out_scale = torch.empty((M, N // 128), dtype=torch.float32, device=a8.device)
        _need(out, torch.float8_e4m3fn, "out")
        if out.shape != (M, N):
            raise OsbError(f"gemm_fp8_blocks: out must be e4m3 [{M}, {N}], got {tuple(out.shape)}")
        b.D8, b.ldd8 = out.data_ptr(), out.stride(0)
        b.d_scale, b.ld_dscale = out_scale.data_ptr(), _scale_view(out_scale, M, N // 128, "out_scale")
    else:
        if out is None:
            out = torch.empty((M, N), dtype=torch.bfloat16, device=a8.device)
        _need(out, torch.bfloat16, "out")
    g = GemmFp8Args()
    g.A, g.W, g.a_scale, g.w_scale = a8.data_ptr(), w8.data_ptr(), a_scale.data_ptr(), w_scale.data_ptr()
    g.bias = bias.data_ptr() if bias is not None else None
    g.D = None if fp8_out else out.data_ptr()
    g.R = residual.data_ptr() if residual is not None else None
    g.gate = gate.data_ptr() if gate is not None else None
    g.mod_index = mod_index.data_ptr() if mod_index is not None else None
    g.M, g.N, g.K = M, N, K
    g.lda, g.ldw, g.ldd = a8.stride(0), w8.stride(0), 0 if fp8_out else out.stride(0)
    g.ldr = residual.stride(0) if residual is not None else 0
    g.group_rows = group_rows if group_rows > 0 else M
    g.gate_stride = gate.stride(0) if gate is not None else 0
    g.epilogue, g.block_n = epilogue, block_n
    with _Timed("gemm_fp8", 2.0 * M * N * K):
        _check(_lib.osb_gemm_fp8_blocks(C.byref(g), C.byref(b), _stream()), "osb_gemm_fp8_blocks")
    return (out, out_scale) if fp8_out else out


def quant_blocks_fp8(x, *, block: int = 128, out=None, out_scale=None):
    """e4m3 quantization of bf16 x [rows, K] (row stride free) with one scale per (row, `block` columns)
    (osb_quant_blocks_fp8): block 128 (one pass) or K (per row, any K; the MLP weights).  Returns (e4m3 [rows, K],
    fp32 [rows, K / block]); `out` / `out_scale` may be column views of wider buffers."""
    import torch

    _need(x, torch.bfloat16, "x")
    if x.dim() != 2:
        raise OsbError(f"quant_blocks_fp8: x must be [rows, K], got {tuple(x.shape)}")
    rows, K = x.shape
    if block <= 0 or K % block:
        raise OsbError(f"quant_blocks_fp8: block {block} does not divide K = {K}")
    if out is None:
        out = torch.empty((rows, K), dtype=torch.float8_e4m3fn, device=x.device)
    if out_scale is None:
        out_scale = torch.empty((rows, K // block), dtype=torch.float32, device=x.device)
    _need(out, torch.float8_e4m3fn, "out")
    if out.shape != (rows, K):
        raise OsbError(f"quant_blocks_fp8: out must be [{rows}, {K}], got {tuple(out.shape)}")
    lds = _scale_view(out_scale, rows, K // block, "out_scale")
    with _Timed("quant_blocks_fp8", 3.0 * rows * K):  # algorithmic bytes: read bf16 + write e4m3
        _check(_lib.osb_quant_blocks_fp8(_ptr(x), x.stride(0), _ptr(out), out.stride(0), _ptr(out_scale), lds, rows, K,
                                         block, _stream()), "osb_quant_blocks_fp8")
    return out, out_scale


def interleave_gated(wi_0, wi_1):
    """[2 d_ff, d_model] weight of the gated-GELU GEMM: row 2c = wi_0[c], row 2c + 1 = wi_1[c]."""
    import torch

    return torch.stack((wi_0, wi_1), dim=1).reshape(2 * wi_0.shape[0], wi_0.shape[1]).contiguous()


def _attn_short_struct(q, k, v, out, *, num_seqs, seqs_per_batch, q_strides, k_strides, Lq, Lk, num_heads, head_dim,
                       kv_lens, q_norm_w, k_norm_w, norm_eps, rope_cos, rope_sin, softmax_scale, q_norm_w2, k_norm_w2,
                       norm_split, impl, rope_half):
    import torch

    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out"), (q_norm_w, "q_norm_w"), (k_norm_w, "k_norm_w")):
        _need(t, torch.bfloat16, n)
    _need(rope_cos, torch.float32, "rope_cos"); _need(rope_sin, torch.float32, "rope_sin")
    _need(kv_lens, torch.int32, "kv_lens")
    a = AttnShortArgs()
    a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.q_ld, a.k_ld, a.v_ld, a.out_ld = q.stride(0), k.stride(0), v.stride(0), out.stride(0)
    a.num_seqs, a.seqs_per_batch = num_seqs, seqs_per_batch
    a.q_batch_stride, a.q_seq_stride, a.q_tok_stride = q_strides
    a.k_batch_stride, a.k_seq_stride, a.k_tok_stride = k_strides
    a.Lq, a.Lk = Lq, Lk
    a.kv_lens = kv_lens.data_ptr() if kv_lens is not None else None
    a.num_heads, a.head_dim = num_heads, head_dim
    a.q_norm_w = q_norm_w.data_ptr() if q_norm_w is not None else None
    a.k_norm_w = k_norm_w.data_ptr() if k_norm_w is not None else None
    a.norm_eps = norm_eps
    a.rope_cos = rope_cos.data_ptr() if rope_cos is not None else None
    a.rope_sin = rope_sin.data_ptr() if rope_sin is not None else None
    a.softmax_scale = softmax_scale if softmax_scale is not None else head_dim ** -0.5
    _need(q_norm_w2, torch.bfloat16, "q_norm_w2"); _need(k_norm_w2, torch.bfloat16, "k_norm_w2")
    a.q_norm_w2 = q_norm_w2.data_ptr() if q_norm_w2 is not None else None
    a.k_norm_w2 = k_norm_w2.data_ptr() if k_norm_w2 is not None else None
    a.norm_split = norm_split
    a.rope_half = int(rope_half)
    a.reserved = impl   # implementation switch of the C ABI; every value runs the one sm_90a kernel
    return a


def attn_short(q, k, v, out, *, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int,
               num_heads: int, head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None, norm_eps: float = 1e-6,
               rope_cos=None, rope_sin=None, softmax_scale: float | None = None, q_norm_w2=None, k_norm_w2=None,
               norm_split: int = 0, impl: int = 0, rope_half: bool = False):
    """softmax(q k^T * scale) v per (sequence, head) with optional fused QK-RMSNorm and RoPE.
    q/k/v/out are 2-D bf16 views [rows, ld]; *_strides = (batch, seq, token) strides in rows."""
    a = _attn_short_struct(q, k, v, out, num_seqs=num_seqs, seqs_per_batch=seqs_per_batch, q_strides=q_strides,
                           k_strides=k_strides, Lq=Lq, Lk=Lk, num_heads=num_heads, head_dim=head_dim, kv_lens=kv_lens,
                           q_norm_w=q_norm_w, k_norm_w=k_norm_w, norm_eps=norm_eps, rope_cos=rope_cos, rope_sin=rope_sin,
                           softmax_scale=softmax_scale, q_norm_w2=q_norm_w2, k_norm_w2=k_norm_w2, norm_split=norm_split,
                           impl=impl, rope_half=rope_half)
    with _Timed("attn_short", 4.0 * num_seqs * Lq * Lk * num_heads * head_dim):  # QK^T + PV FLOPs
        _check(_lib.osb_attn_short(C.byref(a), _stream()), "osb_attn_short")
    return out


def attn_short_bias(q, k, v, out, bias, *, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int,
                    num_heads: int, head_dim: int, kv_lens=None, softmax_scale: float | None = None):
    """attn_short with an additive fp32 bias by relative position (osb_attn_short_bias): the score of query token i and
    key token j is q.k * scale + bias[h, j - i + Lq - 1].  bias fp32 [num_heads, Lq + Lk - 1] (T5's relative attention
    bias) or [Lq + Lk - 1] shared by all heads (0 / -inf: a causal mask)."""
    import torch

    _need(bias, torch.float32, "bias")
    n = Lq + Lk - 1
    if bias is None or not bias.is_contiguous() or bias.shape not in ((n,), (num_heads, n)):
        raise OsbError(f"attn_short_bias: bias must be a contiguous fp32 [{n}] or [{num_heads}, {n}] tensor, got "
                       f"{None if bias is None else tuple(bias.shape)}")
    a = _attn_short_struct(q, k, v, out, num_seqs=num_seqs, seqs_per_batch=seqs_per_batch, q_strides=q_strides,
                           k_strides=k_strides, Lq=Lq, Lk=Lk, num_heads=num_heads, head_dim=head_dim, kv_lens=kv_lens,
                           q_norm_w=None, k_norm_w=None, norm_eps=1e-6, rope_cos=None, rope_sin=None,
                           softmax_scale=softmax_scale, q_norm_w2=None, k_norm_w2=None, norm_split=0, impl=0,
                           rope_half=False)
    with _Timed("attn_short", 4.0 * num_seqs * Lq * Lk * num_heads * head_dim):
        _check(_lib.osb_attn_short_bias(C.byref(a), _ptr(bias), n if bias.dim() == 2 else 0, _stream()),
               "osb_attn_short_bias")
    return out


def attn_frames(q, k, v, *, frame_tokens: int, q_frame0: int = 0, out=None, softmax_scale: float | None = None):
    """Frame-causal attention of one head (osb_attn_frames): q [batch, Lq, D], k / v [batch, Lk, D] bf16, unit stride in
    D, any row stride (column slices of one buffer are fine), k and v with the same batch stride.  Query token i sees key
    j iff j < min(Lk, (q_frame0 + i // frame_tokens + 1) * frame_tokens).  Returns out [batch, Lq, D]."""
    import torch

    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        _need(t, torch.bfloat16, n)
    if q.dim() != 3 or k.dim() != 3 or k.shape != v.shape or q.shape[0] != k.shape[0] or q.shape[2] != k.shape[2]:
        raise OsbError(f"attn_frames: q [batch, Lq, D] and k, v [batch, Lk, D] expected, got {tuple(q.shape)}, "
                       f"{tuple(k.shape)}, {tuple(v.shape)}")
    nb, Lq, D = q.shape
    if out is None:
        out = torch.empty((nb, Lq, D), dtype=q.dtype, device=q.device)
    if out.shape != q.shape:
        raise OsbError(f"attn_frames: out must have q's shape {tuple(q.shape)}, got {tuple(out.shape)}")

    def strides(t, name):
        ld, bs = t.stride(1), t.stride(0)
        if t.shape[1] == 1:
            ld = max(ld, D)
        if nb > 1 and bs % ld:
            raise OsbError(f"attn_frames: the batch stride of {name} ({bs}) is not a multiple of its row stride ({ld})")
        return ld, (bs // ld if nb > 1 else t.shape[1])

    (q_ld, q_bs), (k_ld, k_bs), (v_ld, v_bs), (o_ld, o_bs) = strides(q, "q"), strides(k, "k"), strides(v, "v"), strides(out, "out")
    if nb > 1 and (v_bs != k_bs or o_bs != q_bs):
        raise OsbError("attn_frames: v must have k's batch stride and out q's (in rows)")
    a = AttnFramesArgs()
    a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.q_ld, a.k_ld, a.v_ld, a.out_ld = q_ld, k_ld, v_ld, o_ld
    a.q_batch_stride, a.k_batch_stride = q_bs, k_bs
    a.Lq, a.Lk = Lq, k.shape[1]
    a.batch, a.head_dim, a.frame_tokens, a.q_frame0 = nb, D, frame_tokens, q_frame0
    a.softmax_scale = softmax_scale if softmax_scale is not None else D ** -0.5
    # FLOPs of the visible part only: row i multiplies min(Lk, (q_frame0 + i // hw + 1) hw) keys
    full, rem = divmod(Lq, max(frame_tokens, 1))
    keys = sum(min(k.shape[1], (q_frame0 + f + 1) * frame_tokens) * (frame_tokens if f < full else rem) for f in range(full + (rem > 0)))
    with _Timed("attn_frames", 4.0 * nb * keys * D):
        _check(_lib.osb_attn_frames(C.byref(a), _stream()), "osb_attn_frames")
    return out


# ---- FP8 (e4m3) attention (include/osb200.h, osb_attn_fp8) ------------------------------------------------------------
ATTN_FP8_KEY_BLOCK = 128   # keys per block; the workspace pads L to a multiple of it


class AttnFp8WorkspaceArgs(C.Structure):
    _fields_ = [("q8", C.c_void_p), ("k8", C.c_void_p), ("vt8", C.c_void_p), ("s_q", C.c_void_p), ("s_k", C.c_void_p),
                ("s_v", C.c_void_p), ("v_amax", C.c_void_p), ("capacity_bh", C.c_int64), ("capacity_lpad", C.c_int64)]


class AttnFp8Workspace:
    """Device buffers of `attn_fp8` for B sequences of L tokens and H heads (Lpad = L rounded up to 128): q8 / k8 e4m3
    [B*H, Lpad, 128], vt8 e4m3 [B*H, 128, Lpad] (V transposed, keys permuted inside 32-key groups, include/osb200.h),
    s_q / s_k fp32 [B*H, Lpad], s_v fp32 [B*H, 128] and the zero-initialised v amax scratch [B*H, 128]."""

    def __init__(self, B: int, L: int, H: int, device):
        import torch

        self.B, self.L, self.H = B, L, H
        BH, Lp = B * H, -(-L // ATTN_FP8_KEY_BLOCK) * ATTN_FP8_KEY_BLOCK
        self.Lpad = Lp
        f8 = torch.float8_e4m3fn
        self.q8 = torch.empty(BH, Lp, 128, dtype=f8, device=device)
        self.k8 = torch.empty(BH, Lp, 128, dtype=f8, device=device)
        self.vt8 = torch.empty(BH, 128, Lp, dtype=f8, device=device)
        self.s_q = torch.empty(BH, Lp, dtype=torch.float32, device=device)
        self.s_k = torch.empty(BH, Lp, dtype=torch.float32, device=device)
        self.s_v = torch.empty(BH, 128, dtype=torch.float32, device=device)
        self.v_amax = torch.zeros(BH, 128, dtype=torch.float32, device=device)
        a = self.args = AttnFp8WorkspaceArgs()
        a.q8, a.k8, a.vt8 = self.q8.data_ptr(), self.k8.data_ptr(), self.vt8.data_ptr()
        a.s_q, a.s_k, a.s_v, a.v_amax = self.s_q.data_ptr(), self.s_k.data_ptr(), self.s_v.data_ptr(), self.v_amax.data_ptr()
        a.capacity_bh, a.capacity_lpad = BH, Lp


def attn_fp8_workspace(B: int, L: int, H: int, device) -> AttnFp8Workspace:
    """Allocate the workspace of `attn_fp8` for B sequences of L tokens with H heads of 128."""
    return AttnFp8Workspace(B, L, H, device)


def attn_fp8(q, k, v, out, *, workspace: AttnFp8Workspace, num_seqs: int, seqs_per_batch: int, q_strides, k_strides,
             Lq: int, Lk: int, num_heads: int, head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None,
             norm_eps: float = 1e-6, rope_cos=None, rope_sin=None, softmax_scale: float | None = None, q_norm_w2=None,
             k_norm_w2=None, norm_split: int = 0, impl: int = 0, rope_half: bool = False):
    """`attn_short` on e4m3 operands (osb_attn_fp8): q / k quantized per (token, head) after QK-norm and RoPE, v per
    channel, P as e4m3(256 p).  Self-attention of one sequence per batch element with heads of 128 (Lq == Lk,
    seqs_per_batch == 1, no kv_lens); the keywords are those of `attn_short`.  `workspace` (attn_fp8_workspace) must
    hold num_seqs * num_heads sequence-heads of Lq tokens; after the call it holds the quantized operands."""
    if not isinstance(workspace, AttnFp8Workspace):
        raise OsbError("attn_fp8: workspace must come from attn_fp8_workspace()")
    a = _attn_short_struct(q, k, v, out, num_seqs=num_seqs, seqs_per_batch=seqs_per_batch, q_strides=q_strides,
                           k_strides=k_strides, Lq=Lq, Lk=Lk, num_heads=num_heads, head_dim=head_dim, kv_lens=kv_lens,
                           q_norm_w=q_norm_w, k_norm_w=k_norm_w, norm_eps=norm_eps, rope_cos=rope_cos, rope_sin=rope_sin,
                           softmax_scale=softmax_scale, q_norm_w2=q_norm_w2, k_norm_w2=k_norm_w2, norm_split=norm_split,
                           impl=impl, rope_half=rope_half)
    if workspace.q8.device != q.device:
        raise OsbError(f"attn_fp8: the workspace is on {workspace.q8.device}, q on {q.device}")
    with _Timed("attn_fp8", 4.0 * num_seqs * Lq * Lk * num_heads * head_dim):  # QK^T + PV FLOPs
        _check(_lib.osb_attn_fp8(C.byref(a), C.byref(workspace.args), _stream()), "osb_attn_fp8")
    return out


# ---- head tiles: projection GEMM -> attention without a layout pass (include/osb200.h) ------------------------------
class TileMap(C.Structure):
    _fields_ = [("mode", C.c_int32), ("L", C.c_int32), ("S", C.c_int32), ("T", C.c_int32), ("G", C.c_int32),
                ("tps", C.c_int32), ("tile_rows", C.c_int32), ("reserved", C.c_int32)]

    def key(self):
        return (self.mode, self.L, self.S, self.T, self.G, self.tps, self.tile_rows)


class HeadTilesArgs(C.Structure):
    _fields_ = [
        ("tiles", C.c_void_p), ("kind_stride", C.c_int64), ("head_stride", C.c_int64), ("map", TileMap),
        ("num_heads", C.c_int32), ("head_dim", C.c_int32), ("nkinds", C.c_int32),
        ("norm_mask", C.c_uint32), ("rope_mask", C.c_uint32), ("reserved", C.c_int32),
        ("norm_w", C.c_void_p * 4), ("norm_eps", C.c_float), ("reserved2", C.c_int32),
        ("rope_cos", C.c_void_p), ("rope_sin", C.c_void_p),
    ]


class AttnTilesArgs(C.Structure):
    _fields_ = [
        ("q_tiles", C.c_void_p), ("k_tiles", C.c_void_p), ("v_tiles", C.c_void_p),
        ("q_head_stride", C.c_int64), ("kv_head_stride", C.c_int64), ("q_map", TileMap),
        ("kv_tile_rows", C.c_int32), ("kv_tiles_per_set", C.c_int32), ("Lk", C.c_int32),
        ("num_heads", C.c_int32), ("head_dim", C.c_int32), ("reserved", C.c_int32),
        ("num_seqs", C.c_int64), ("kv_lens", C.c_void_p), ("out", C.c_void_p), ("out_ld", C.c_int64),
        ("softmax_scale", C.c_float), ("reserved2", C.c_int32), ("out_scatter", C.c_void_p),
    ]


def tile_map(mode: int, L: int, S: int = 0, T: int = 0, *, keys_only: bool = False, pack: bool = True) -> TileMap:
    """Token row -> (tile, row) map of include/osb200.h `osb_tile_map`.  mode 0: sequences are contiguous blocks of L
    rows; mode 1: sequences run along T of a frame-major [B, T, S] token stream (L == T).  Short sequences (L <= 64) are
    packed 128 // L per tile (self-attention: a tile is its own key set; `pack=False` for cross-attention queries,
    whose key set is per sequence); `keys_only` (text keys of cross-attention) never packs either."""
    m = TileMap()
    m.mode, m.L, m.S, m.T = mode, L, S, T
    if L <= 64 and pack and not keys_only:
        m.G, m.tps = 128 // L, 1
        m.tile_rows = -(-(m.G * L) // 16) * 16
    else:
        m.G = 1
        n = -(-L // 128)
        # (keys-only tiles used to be balanced, 300 -> 3 x 112; a 112-row tile ends in the middle of a 32-column softmax
        # chunk and sent a quarter of the chunks through the per-element masked path: full 128-row tiles + a short last one)
        m.tile_rows = 128 if L > 128 else -(-(-(-L // n)) // 16) * 16
        m.tps = -(-L // m.tile_rows)
    return m


class HeadTiles:
    """A buffer of head tiles: `kinds` column groups (q | k | v ...) x heads x tiles.  Zero-initialised: rows no token
    maps to (ragged last tile, head-dim tail) must stay finite, they are multiplied by P = 0 in the PV product."""

    def __init__(self, rows: int, tmap: TileMap, kinds: int, heads: int, head_dim: int, device):
        import torch

        self.rows, self.map, self.kinds, self.heads, self.head_dim = rows, tmap, kinds, heads, head_dim
        self.tiles_per_head = int(_lib.osb_head_tiles_per_head(C.byref(tmap), rows))
        if self.tiles_per_head <= 0:
            raise OsbError(f"tile map {tmap.key()} does not fit {rows} rows")
        self.tile_bytes = tmap.tile_rows * (-(-head_dim // 16) * 16) * 2
        self.head_stride = self.tiles_per_head * self.tile_bytes
        self.kind_stride = heads * self.head_stride
        self.buf = torch.zeros(kinds * self.kind_stride, dtype=torch.uint8, device=device)

    def kind_ptr(self, kind: int) -> int:
        return self.buf.data_ptr() + kind * self.kind_stride


def gemm_head_tiles(a, w, bias, tiles: HeadTiles, *, nkinds: int, norm_w=(), rope=None, rope_kinds: int = 0,
                    eps: float = 1e-6, kind0: int = 0, general: bool = False):
    """tiles[kind0 + n // C] = head_tiles(a @ w.T + bias): each output row is split into heads; kinds listed in
    `norm_w` (bf16 [D] or None per kind) get per-head RMSNorm, kinds in the `rope_kinds` bit mask get interleaved-pair
    RoPE by token position from `rope` = (cos, sin) fp32 [L, D/2]; one rounding to bf16 at the row's place in its tile."""
    import torch

    _need(a, torch.bfloat16, "a"); _need(w, torch.bfloat16, "w"); _need(bias, torch.bfloat16, "bias")
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] == w.shape[1]
    M, K = a.shape
    N = w.shape[0]
    Cc = tiles.heads * tiles.head_dim
    assert M == tiles.rows and N % Cc == 0 and kind0 + N // Cc <= tiles.kinds
    g = GemmArgs()
    g.A, g.W, g.bias = a.data_ptr(), w.data_ptr(), (bias.data_ptr() if bias is not None else None)
    g.M, g.N, g.K = M, N, K
    g.lda, g.ldw = a.stride(0), w.stride(0)
    t = HeadTilesArgs()
    t.tiles = tiles.kind_ptr(kind0)
    t.kind_stride, t.head_stride, t.map = tiles.kind_stride, tiles.head_stride, tiles.map
    t.num_heads, t.head_dim, t.nkinds = tiles.heads, tiles.head_dim, nkinds
    t.reserved = 1 if general else 0   # force the general per-row-store epilogue (tests / A-B)
    mask = 0
    for i, nw in enumerate(norm_w):
        if nw is not None:
            _need(nw, torch.bfloat16, "norm_w")
            t.norm_w[i] = nw.data_ptr()
            mask |= 1 << i
    t.norm_mask, t.rope_mask, t.norm_eps = mask, (rope_kinds if rope is not None else 0), eps
    if rope is not None:
        _need(rope[0], torch.float32, "rope cos"); _need(rope[1], torch.float32, "rope sin")
        t.rope_cos, t.rope_sin = rope[0].data_ptr(), rope[1].data_ptr()
    with _Timed("gemm", 2.0 * M * N * K):
        _check(_lib.osb_gemm_head_tiles(C.byref(g), C.byref(t), _stream()), "osb_gemm_head_tiles")
    return tiles


def attn_tiles(q: HeadTiles, kv: HeadTiles, out, *, q_kind: int = 0, k_kind: int = 1, v_kind: int = 2, Lk: int,
               num_seqs: int, kv_lens=None, softmax_scale: float | None = None, out_scatter: Scatter | None = None,
               out_ld: int | None = None, out_map: TileMap | None = None):
    """out = softmax(q k^T * scale) v per (sequence, head) over head tiles (osb_attn_tiles).  Self-attention: q and kv
    are the same buffer (kinds 0, 1, 2); cross-attention: kv holds the text keys / values (`keys_only` map).
    `out_map`: the token order of `out` when it differs from the order the q tiles were written from (temporal attention:
    tiles from the transposed [B, S, T] stream (mode 0), output rows frame-major (mode 1))."""
    a = _attn_tiles_struct(q, kv, out, Lk=Lk, num_seqs=num_seqs, kv_lens=kv_lens, softmax_scale=softmax_scale,
                           out_scatter=out_scatter, out_ld=out_ld, out_map=out_map, who="attn_tiles")
    a.q_tiles, a.k_tiles, a.v_tiles = q.kind_ptr(q_kind), kv.kind_ptr(k_kind), kv.kind_ptr(v_kind)
    a.q_head_stride, a.kv_head_stride = q.head_stride, kv.head_stride
    with _Timed("attn_tiles", 4.0 * num_seqs * q.map.L * Lk * q.heads * q.head_dim):
        _check(_lib.osb_attn_tiles(C.byref(a), _stream()), "osb_attn_tiles")
    return out


def _attn_tiles_struct(q, kv, out, *, Lk, num_seqs, kv_lens, softmax_scale, out_scatter, out_ld, out_map, who):
    """osb_attn_tiles_args without the tile pointers: maps, key sets and output routing (shared by the bf16 and the FP8
    tile attention)."""
    import torch

    _need(out, torch.bfloat16, "out"); _need(kv_lens, torch.int32, "kv_lens")
    assert (out is None) != (out_scatter is None), "exactly one of out / out_scatter"
    if kv_lens is not None and q.map.G > 1:   # the kernel reads kv_lens for unpacked query maps only
        raise OsbError(f"{who}: kv_lens applies to unpacked query maps only (G == 1); packed sequences see all Lk keys")
    a = AttnTilesArgs()
    if out_map is not None:   # output rows in another order than the rows the tiles were written from (same tiling)
        assert out_map.key()[4:] == q.map.key()[4:] and out_map.L == q.map.L
    a.q_map = out_map if out_map is not None else q.map
    a.kv_tile_rows = kv.map.tile_rows
    a.kv_tiles_per_set = kv.map.tps
    a.Lk, a.num_heads, a.head_dim = Lk, q.heads, q.head_dim
    a.num_seqs = num_seqs
    a.kv_lens = kv_lens.data_ptr() if kv_lens is not None else None
    if out_scatter is not None:   # rows go to peer buffers (row stride out_ld elements on every destination)
        a.out, a.out_ld = None, int(out_ld)
        a.out_scatter = C.addressof(out_scatter)
    else:
        a.out, a.out_ld = out.data_ptr(), out.stride(0)
    a.softmax_scale = softmax_scale if softmax_scale is not None else q.head_dim ** -0.5
    return a


# ---- FP8 (e4m3) head tiles (include/osb200.h, osb_head_tiles_fp8 / osb_attn_tiles_fp8) ---------------------------------
TILE_FP8_BYTES = 128 * 128   # one e4m3 tile: 128 rows of 128 bytes, 128-byte swizzle
TILE_FP8_SCALES = 128        # fp32 scales per tile (per row for q / k, per channel for v)


class TilesFp8(C.Structure):
    _fields_ = [("codes", C.c_void_p), ("scales", C.c_void_p), ("tiles_per_head", C.c_int64), ("num_heads", C.c_int32),
                ("reserved", C.c_int32)]


class HeadTilesFp8Args(C.Structure):
    _fields_ = [
        ("tiles", C.c_void_p), ("kind_stride", C.c_int64), ("head_stride", C.c_int64), ("dst", TilesFp8),
        ("tile_rows", C.c_int32), ("head_dim", C.c_int32), ("nkinds", C.c_int32), ("v_period", C.c_int32),
        ("v_slot", C.c_int32), ("reserved", C.c_int32),
    ]


class AttnTilesFp8Operands(C.Structure):
    _fields_ = [("q8", C.c_void_p), ("k8", C.c_void_p), ("v8", C.c_void_p), ("s_q", C.c_void_p), ("s_k", C.c_void_p),
                ("s_v", C.c_void_p), ("q_head_tiles", C.c_int64), ("kv_head_tiles", C.c_int64)]


class HeadTilesFp8:
    """The e4m3 twin of a HeadTiles buffer: the same kinds x heads x tiles, each tile 128 rows x 128 bytes of codes
    (`codes`, uint8 [kinds, heads, tiles, 128, 128] in the 128-byte swizzle) and 128 fp32 scales (`scales`, [kinds, heads,
    tiles, 128]).  Zero-filled once, like HeadTiles."""

    def __init__(self, tiles: HeadTiles):
        import torch

        if tiles.head_dim not in (64, 72):
            raise OsbError(f"FP8 head tiles are built for head_dim 64 and 72, not {tiles.head_dim}")
        self.src, self.map, self.kinds, self.heads, self.head_dim = tiles, tiles.map, tiles.kinds, tiles.heads, tiles.head_dim
        self.tiles_per_head = tiles.tiles_per_head
        n = tiles.kinds * tiles.heads * tiles.tiles_per_head
        dev = tiles.buf.device
        self.codes = torch.zeros(tiles.kinds, tiles.heads, tiles.tiles_per_head, 128, 128, dtype=torch.uint8, device=dev)
        self.scales = torch.zeros(tiles.kinds, tiles.heads, tiles.tiles_per_head, TILE_FP8_SCALES, dtype=torch.float32,
                                  device=dev)
        assert self.codes.numel() == n * TILE_FP8_BYTES

    def codes_ptr(self, kind: int) -> int:
        return self.codes[kind].data_ptr()

    def scales_ptr(self, kind: int) -> int:
        return self.scales[kind].data_ptr()


def head_tiles_fp8(tiles: HeadTiles, dst: HeadTilesFp8, *, kind0: int = 0, nkinds: int | None = None, v_period: int = 0,
                   v_slot: int = 0) -> HeadTilesFp8:
    """dst[kind0 + k] = e4m3(tiles[kind0 + k]) for k < nkinds, in one launch (osb_head_tiles_fp8): kind k (counted from
    kind0) is converted as a value kind (transposed, per-channel scales) iff v_period > 0 and k % v_period == v_slot,
    else as a query / key kind (per-row scales)."""
    if dst.src is not tiles:
        raise OsbError("head_tiles_fp8: dst must be HeadTilesFp8(tiles) of the same bf16 tiles")
    nkinds = tiles.kinds - kind0 if nkinds is None else nkinds
    if not (0 <= kind0 and nkinds >= 1 and kind0 + nkinds <= tiles.kinds):
        raise OsbError(f"head_tiles_fp8: kinds [{kind0}, {kind0 + nkinds}) outside the {tiles.kinds} of the buffer")
    a = HeadTilesFp8Args()
    a.tiles, a.kind_stride, a.head_stride = tiles.kind_ptr(kind0), tiles.kind_stride, tiles.head_stride
    a.dst.codes, a.dst.scales = dst.codes_ptr(kind0), dst.scales_ptr(kind0)
    a.dst.tiles_per_head, a.dst.num_heads = dst.tiles_per_head, dst.heads
    a.tile_rows, a.head_dim, a.nkinds, a.v_period, a.v_slot = tiles.map.tile_rows, tiles.head_dim, nkinds, v_period, v_slot
    with _Timed("head_tiles_fp8", float(nkinds * tiles.heads * tiles.tiles_per_head * (tiles.tile_bytes + TILE_FP8_BYTES))):
        _check(_lib.osb_head_tiles_fp8(C.byref(a), _stream()), "osb_head_tiles_fp8")
    return dst


def attn_tiles_fp8(q: HeadTilesFp8, kv: HeadTilesFp8, out, *, q_kind: int = 0, k_kind: int = 1, v_kind: int = 2, Lk: int,
                   num_seqs: int, kv_lens=None, softmax_scale: float | None = None, out_scatter: Scatter | None = None,
                   out_ld: int | None = None, out_map: TileMap | None = None):
    """`attn_tiles` on e4m3 head tiles (osb_attn_tiles_fp8): the same keywords and set shapes, operands from
    head_tiles_fp8.  head_dim 64 or 72."""
    if not isinstance(q, HeadTilesFp8) or not isinstance(kv, HeadTilesFp8):
        raise OsbError("attn_tiles_fp8: q and kv must be HeadTilesFp8 buffers")
    a = _attn_tiles_struct(q, kv, out, Lk=Lk, num_seqs=num_seqs, kv_lens=kv_lens, softmax_scale=softmax_scale,
                           out_scatter=out_scatter, out_ld=out_ld, out_map=out_map, who="attn_tiles_fp8")
    o = AttnTilesFp8Operands()
    o.q8, o.k8, o.v8 = q.codes_ptr(q_kind), kv.codes_ptr(k_kind), kv.codes_ptr(v_kind)
    o.s_q, o.s_k, o.s_v = q.scales_ptr(q_kind), kv.scales_ptr(k_kind), kv.scales_ptr(v_kind)
    o.q_head_tiles, o.kv_head_tiles = q.tiles_per_head, kv.tiles_per_head
    with _Timed("attn_tiles_fp8", 4.0 * num_seqs * q.map.L * Lk * q.heads * q.head_dim):
        _check(_lib.osb_attn_tiles_fp8(C.byref(a), C.byref(o), _stream()), "osb_attn_tiles_fp8")
    return out


def tmap_cache_stats():
    h, m = C.c_int64(0), C.c_int64(0)
    _lib.osb_tmap_cache_stats(C.byref(h), C.byref(m))
    return int(h.value), int(m.value)


# ---- causal 3D VAE ops (NDHWC) -------------------------------------------------------------------------
def group_stats(x, groups: int, eps: float = 1e-6):
    """GroupNorm statistics of x bf16 [nb, T, H, W, C] (channels last) -> fp32 [nb, groups, 2] = (mean, rstd)."""
    import torch

    _need(x, torch.bfloat16, "x")
    assert x.dim() == 5 and x.is_contiguous()
    nb, Cc = x.shape[0], x.shape[-1]
    pos = x.shape[1] * x.shape[2] * x.shape[3]
    ws_bytes = int(_lib.osb_group_stats_workspace_bytes(nb, pos, groups))
    ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=x.device)
    out = torch.empty(nb, groups, 2, dtype=torch.float32, device=x.device)
    with _Timed("group_stats", 2.0 * x.numel()):  # algorithmic bytes: one read
        _check(_lib.osb_group_stats(_ptr(x), nb, pos, Cc, groups, eps, _ptr(ws), ws_bytes, _ptr(out), _stream()),
               "osb_group_stats")
    return out


def vae_prep(x, *, stats=None, gamma=None, beta=None, groups: int = 32, silu: bool = False, up=(1, 1, 1),
             pad=(0, 0, 0), cp: int | None = None, slack_bytes: int = 128):
    """[GroupNorm-apply + SiLU] + nearest upsample + replicate pad of x bf16 [nb,T,H,W,C] -> padded bf16
    [nb,Tp,Hp,Wp,cp] (one pass).  pad = (front frames, rows each side, cols each side)."""
    import torch

    _need(x, torch.bfloat16, "x"); _need(stats, torch.float32, "stats")
    _need(gamma, torch.bfloat16, "gamma"); _need(beta, torch.bfloat16, "beta")
    assert x.dim() == 5 and x.is_contiguous()
    nb, T, H, W, Cc = x.shape
    cp = cp or Cc
    tu = T if up[0] == 1 else 1 + up[0] * (T - 1)
    tp, hp, wp = tu + pad[0], H * up[1] + 2 * pad[1], W * up[2] + 2 * pad[2]
    n = nb * tp * hp * wp * cp
    buf = torch.empty(n + slack_bytes // 2, dtype=torch.bfloat16, device=x.device)  # slack: narrow-mode windows
    if slack_bytes:
        buf[n:].zero_()
    y = buf[:n].view(nb, tp, hp, wp, cp)
    a = VaePrepArgs()
    a.x, a.y = x.data_ptr(), y.data_ptr()
    a.mean_rstd = stats.data_ptr() if stats is not None else None
    a.gamma = gamma.data_ptr() if gamma is not None else None
    a.beta = beta.data_ptr() if beta is not None else None
    a.nb, a.t, a.h, a.w, a.c = nb, T, H, W, Cc
    a.groups, a.silu = groups, int(silu)
    a.ft, a.fh, a.fw = up
    a.pad_t, a.pad_h, a.pad_w = pad
    a.cp = cp
    with _Timed("vae_prep", 2.0 * (x.numel() + n)):
        _check(_lib.osb_vae_prep(C.byref(a), _stream()), "osb_vae_prep")
    return y


def conv3d(x_pad, w_packed, bias, *, out_thw, stride=(1, 1, 1), taps=(3, 3, 3), narrow: bool = False, residual=None,
           block_n: int = 0):
    """y = conv3d(x_pad) + bias (+ residual): x_pad bf16 [nb,Tp,Hp,Wp,Cp] (already padded), w_packed bf16 [Cout, K]
    (see pack_conv_weight), y bf16 [nb, T_out, H_out, W_out, Cout]."""
    import torch

    _need(x_pad, torch.bfloat16, "x_pad"); _need(w_packed, torch.bfloat16, "w_packed"); _need(bias, torch.bfloat16, "bias")
    _need(residual, torch.bfloat16, "residual")
    nb, tp, hp, wp, cp = x_pad.shape
    cout = w_packed.shape[0]
    y = torch.empty(nb, *out_thw, cout, dtype=torch.bfloat16, device=x_pad.device)
    a = Conv3dArgs()
    a.x_pad, a.w, a.y = x_pad.data_ptr(), w_packed.data_ptr(), y.data_ptr()
    a.bias = bias.data_ptr() if bias is not None else None
    a.residual = residual.data_ptr() if residual is not None else None
    a.nb, a.tp, a.hp, a.wp, a.cp = nb, tp, hp, wp, cp
    a.t_out, a.h_out, a.w_out = out_thw
    a.cout = cout
    a.st, a.sh, a.sw = stride
    a.kt, a.kh, a.kw = taps
    a.narrow, a.block_n = int(narrow), block_n
    with _Timed("conv3d", 2.0 * y.numel() * w_packed.shape[1]):  # MACs incl. K padding (algorithmic count is the caller's)
        _check(_lib.osb_conv3d_ndhwc(C.byref(a), _stream()), "osb_conv3d_ndhwc")
    return y


def pack_conv_weight(w, cp: int, narrow: bool, cout_pad: int | None = None):
    """torch Conv3d weight [Cout, Cin, kt, kh, kw] -> bf16 [Cout_p, K] K-major in the order the kernel walks K
    (include/osb200.h osb_conv3d_args.w).  Done once at load time."""
    import torch

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
    """out = x + dt * (uncond2 + g_img*(uncond - uncond2) + g_txt*(cond - uncond)); bf16 tensors of one shape."""
    import torch

    for t, n in ((cond, "cond"), (uncond, "uncond"), (uncond2, "uncond2"), (x, "x"), (g_img_map, "g_img_map")):
        _need(t, torch.bfloat16, n)
        assert t is None or t.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    n = x.numel()
    with _Timed("cfg_euler", 2.0 * n * (5 if uncond2 is not None else 4)):
        _check(_lib.osb_cfg_euler(_ptr(cond), _ptr(uncond), _ptr(uncond2), _ptr(x), _ptr(out), n, g_txt, g_img,
                                  _ptr(g_img_map), g_img_map.numel() if g_img_map is not None else 0, dt, _stream()),
               "osb_cfg_euler")
    return out


def rf_masked_step(vc, vu, z, frame_mask, t_cur, t_next, *, guidance: float, noise=None, update: bool = True,
                   num_timesteps: int = 1000, out=None):
    """The frame-masked rectified-flow step (osb_rf_masked_step): z bf16 [B, C, T, H, W]; frame_mask fp32 [B, T] (1 =
    generate, 0 = keep, in between = edit ratio); t_cur / t_next fp32 [B] on the device.  Frames with frame_mask * N >=
    t_cur get z + (t_cur - t_next) / N * (vu + guidance (vc - vu)), the rest keep z bit for bit; with `noise`, frames that
    reach t_next for the first time are then re-noised to (1 - t_next/N) z + (t_next/N) noise.  update=False is the
    prologue before the first model call (re-noise only, vc / vu unused; "first time" = frame_mask != 1).  out may be z."""
    import torch

    for t, n in ((vc, "vc"), (vu, "vu"), (z, "z"), (noise, "noise"), (out, "out")):
        _need(t, torch.bfloat16, n)
        if t is not None and (t.shape != z.shape or not t.is_contiguous()):
            raise OsbError(f"{n} must be a contiguous tensor of the latent's shape {tuple(z.shape)}")
    for t, n in ((frame_mask, "frame_mask"), (t_cur, "t_cur"), (t_next, "t_next")):
        _need(t, torch.float32, n)
        if not t.is_contiguous():
            raise OsbError(f"{n} must be contiguous")
    if z.dim() != 5:
        raise OsbError("z must be [B, C, T, H, W]")
    B, Cc, T, H, W = z.shape
    if frame_mask.shape != (B, T) or t_cur.shape != (B,) or t_next.shape != (B,):
        raise OsbError(f"frame_mask must be [B, T] = [{B}, {T}] and t_cur / t_next [B]")
    if out is None:
        out = torch.empty_like(z)
    n = z.numel()
    with _Timed("rf_masked_step", 2.0 * n * (2 + 2 * int(update) + int(noise is not None))):  # dense bytes: all frames
        _check(_lib.osb_rf_masked_step(_ptr(vc), _ptr(vu), _ptr(z), _ptr(noise), _ptr(out), _ptr(frame_mask), _ptr(t_cur),
                                       _ptr(t_next), B, Cc, T, H * W, guidance, num_timesteps, int(update), _stream()),
               "osb_rf_masked_step")
    return out
