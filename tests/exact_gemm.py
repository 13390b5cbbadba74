"""GEMM cases whose arithmetic is exact in every format the kernels use, for bit-identical tests of `gemm`, `gemm_lora`
(with and without DoRA's col_scale), `gemm_fp8` and `gemm_fp8_blocks` (with its FP8-emitting GELU epilogue).

A rel-L2 bound cannot see an error confined to a few elements (one ragged column tile, one k-block's scale).  These
operands remove the rounding instead of bounding it:
  - bf16 A, U, W, B are {0, +-1} x a power of two per row (2^-2 .. 2^2); e4m3 A codes are {0, +-1}, W codes {0, +-1, +-2};
  - FP8 scales are powers of two in [2^-3, 2^3], DoRA's col_scale in [2^-1, 2^2], gates +-{0.5, 1, 2};
  - bias and residual are bf16 multiples of 2^-2 with magnitude <= 64.
Every product is then exact, every partial sum is a small multiple of a power of two, and every scale, gate and
col_scale step is a power-of-two multiply.  `check_budget` proves in fp64 that each value stays within 22 significant
bits (fp32 has 24) and each FP8 k-block partial is an integer of magnitude <= 256, so the kernel's fp32 result is one
value whatever its summation order, and its one rounding to bf16 must equal the fp64 reference rounded once, bit for
bit.  Exponents and signs vary by row, column and k-block, so a permuted, shifted or dropped row, column, k-block or
scale changes the result.

The GELU epilogues are exact only where GELU is the identity: with unit-magnitude operands, K <= 3072 and a bias of 4096
every pre-activation v lies in [1024, 7168], where gelu_tanh(v) = 0.5 v (1 + tanh(u)) = v once tanh saturates to 1.0.
The FP8 GELU epilogue's block scale fp32(amax / 448) and codes e4m3_rn(v / s) then follow from torch's fp32 IEEE
division and float8_e4m3fn cast.

Generators build on `device` from a seeded generator on that device, so a GPU test never materialises its large
operands on the host."""
import math

import torch

E4M3 = torch.float8_e4m3fn
EPI_BIAS, EPI_BIAS_GELU_TANH, EPI_BIAS_GATE_RES, EPI_BIAS_GELU_TANH_FP8 = 0, 1, 2, 5
EPI_NAMES = {EPI_BIAS: "bias", EPI_BIAS_GELU_TANH: "gelu", EPI_BIAS_GATE_RES: "gate_res", EPI_BIAS_GELU_TANH_FP8: "gelu_fp8"}
FP8_PARTIAL_MAX = 256     # integer k-block partials up to this magnitude are exact in the FP8 tensor core
FP32_BITS = 22            # significant bits allowed for a value the kernel forms in fp32 (2 bits under fp32's 24)
GELU_FLOOR = 1024.0       # pre-activations at or above this make gelu_tanh the identity (tanh saturated)
GELU_BIAS = 4096.0
PAD = 32                  # extra columns around sliced operands and outputs


class BudgetError(AssertionError):
    pass


# ---- exactness analysis (fp64) ----------------------------------------------------------------------------------------
def _grid(x):
    """Per element: the largest power of two that x is a multiple of (inf for 0).  x fp64."""
    m, e = torch.frexp(x)
    mi = (m * 2.0 ** 53).to(torch.int64)                  # odd part times a power of two, exact
    low = (mi & -mi).to(torch.float64)
    return torch.where(x == 0, torch.full_like(x, math.inf), torch.ldexp(low, e - 53))


def _row_grid(x):
    return _grid(x).amin(-1)


def _pow2(name, x, lo, hi):
    x = x.double()
    m, _ = torch.frexp(x.abs())
    if not bool(((m == 0.5) & (x.abs() >= lo) & (x.abs() <= hi)).all()):
        raise BudgetError(f"{name}: every value must be +-2^e with 2^e in [{lo}, {hi}]")


def _fits(step, grid, bound):
    """grid: power of two every term is a multiple of; bound: largest magnitude any partial value can take."""
    grid, bound = torch.broadcast_tensors(grid, bound)
    live = torch.isfinite(grid) & (bound > 0)
    if not bool(live.any()):
        return
    bits = float((torch.log2(bound[live]) - torch.log2(grid[live])).max())
    if bits > FP32_BITS:
        raise BudgetError(f"{step}: a value may need {bits:.2f} significant bits (budget {FP32_BITS}): not exact in fp32")


def _gate_rows(case):
    M = case.M
    g = torch.arange(M, device=case.gate.device) // (case.group_rows if case.group_rows > 0 else M)
    if case.mod_index is not None:
        g = case.mod_index.long()[g]
    return case.gate.double()[g]


def check_budget(case):
    """Proves in fp64, before anything runs, that every value the kernel forms before its one rounding is exact:
    FP8 k-block partials are integers of magnitude <= 256 (the tensor core's own accumulation), and the bf16 wgmma
    accumulator over all of K, the fp32 accumulator over the k-blocks and each epilogue step (scale, bias, gate,
    residual) need at most FP32_BITS significant bits.  Raises BudgetError naming the step that does not fit."""
    d = lambda t: None if t is None else t.detach().double()  # noqa: E731
    if case.fn in ("gemm", "gemm_lora"):
        a, w = d(case.a), d(case.w)
        grid = _row_grid(a)[:, None] * _row_grid(w)[None]
        bound = torch.minimum(a.abs().sum(1)[:, None] * w.abs().amax(1)[None],
                              a.abs().amax(1)[:, None] * w.abs().sum(1)[None])
        if case.u is not None:
            u, b = d(case.u), d(case.b)
            grid = torch.minimum(grid, _row_grid(u)[:, None] * _row_grid(b)[None])
            bound = bound + u.abs().sum(1)[:, None] * b.abs().amax(1)[None]
        _fits("bf16 accumulator", grid, bound)
        if case.col_scale is not None:
            cs = d(case.col_scale)
            _pow2("col_scale", cs, 2.0 ** -1, 2.0 ** 2)
            grid, bound = grid * cs[None], bound * cs[None]
            _fits("col_scale", grid, bound)
    else:
        a, w = d(case.a8), d(case.w8)
        if not (bool((a == a.round()).all()) and bool((w == w.round()).all())):
            raise BudgetError("FP8 codes must be integers")
        M, K = a.shape
        KB = K // 128
        part = a.abs().view(M, KB, 128).sum(-1)            # [M, KB]: sum |a| over each k-block
        wmax = w.abs().amax(1)                             # [N]
        p = float(part.max()) * float(wmax.max())
        if p > FP8_PARTIAL_MAX:
            raise BudgetError(f"FP8 k-block partial: an integer partial may reach {p:g} > {FP8_PARTIAL_MAX}")
        sa, sw = d(case.a_scale), d(case.w_scale)
        _pow2("a_scale", sa, 2.0 ** -3, 2.0 ** 3)
        _pow2("w_scale", sw, 2.0 ** -3, 2.0 ** 3)
        if case.fn == "gemm_fp8_blocks" and (sa.dim() == 2 or case.epilogue == EPI_BIAS_GELU_TANH_FP8):
            # each k-block partial is scaled by a_scale[m, kb] as it is added into the fp32 accumulator
            sa2 = sa if sa.dim() == 2 else sa[:, None].expand(M, KB)
            grid = sa2.amin(1)[:, None]
            bound = (sa2 * part).sum(1)[:, None] * wmax[None]
            _fits("fp32 accumulator over the k-blocks", grid, bound)
            grid, bound = grid * sw[None], bound * sw[None]
        else:
            # integer partials summed in fp32, then one multiply by a_scale[m] * w_scale[n]
            grid = torch.ones(M, 1, dtype=torch.float64, device=a.device)
            bound = part.sum(1)[:, None] * wmax[None]
            _fits("fp32 accumulator over the k-blocks", grid, bound)
            grid, bound = grid * sa[:, None] * sw[None], bound * sa[:, None] * sw[None]
    acc_bound = bound
    if case.bias is not None:
        bias = d(case.bias)
        grid = torch.minimum(grid, _grid(bias)[None])
        bound = bound + bias.abs()[None]
        _fits("bias", grid, bound)
    if case.epilogue in (EPI_BIAS_GELU_TANH, EPI_BIAS_GELU_TANH_FP8):
        low = (d(case.bias)[None] if case.bias is not None else 0.0) - acc_bound
        if float(low.min()) < GELU_FLOOR:
            raise BudgetError(f"GELU regime: a pre-activation may fall to {float(low.min()):g} < {GELU_FLOOR:g}, where "
                              "gelu_tanh is not the identity")
    elif case.epilogue == EPI_BIAS_GATE_RES:
        if case.gate is not None:
            g = _gate_rows(case)
            _pow2("gate", g, 0.5, 2.0)
            grid, bound = grid * g.abs(), bound * g.abs()
            _fits("gate", grid, bound)
        if case.residual is not None:
            r = d(case.residual)
            grid = torch.minimum(grid, _grid(r))
            bound = bound + r.abs()
            _fits("residual", grid, bound)


def reference(case):
    """The fp64 value of the call before its one rounding: exact, given check_budget."""
    if case.fn in ("gemm", "gemm_lora"):
        acc = case.a.double() @ case.w.double().t()
        if case.u is not None:
            acc = acc + case.u.double() @ case.b.double().t()
        if case.col_scale is not None:
            acc = acc * case.col_scale.double()[None]
    else:
        sa = case.a_scale.double()
        a = case.a8.double() * (sa.repeat_interleave(128, 1) if sa.dim() == 2 else sa[:, None])
        acc = (a @ case.w8.double().t()) * case.w_scale.double()[None]
    if case.bias is not None:
        acc = acc + case.bias.double()[None]
    if case.epilogue == EPI_BIAS_GATE_RES:
        if case.gate is not None:
            acc = acc * _gate_rows(case)
        if case.residual is not None:
            acc = acc + case.residual.double()
    return acc        # GELU: the identity in the regime check_budget enforces


def fp8_gelu_expected(v):
    """FP8 GELU epilogue of an exact fp64 value v [M, N] (gelu = identity): (e4m3 codes, fp32 scales [M, N / 128])."""
    M, N = v.shape
    x = v.float().view(M, N // 128, 128)                # exact: check_budget bounds v to fp32's significand
    amax = x.abs().amax(-1)
    # a tensor divisor: torch on CUDA divides by a Python scalar as a multiply by its (rounded) reciprocal, which is not
    # the IEEE quotient the kernel computes
    s = torch.where(amax > 0, amax / torch.full_like(amax, 448.0), torch.ones_like(amax))
    return (x / s[..., None]).clamp(-448.0, 448.0).to(E4M3).view(M, N), s


# ---- operands ---------------------------------------------------------------------------------------------------------
def _ints(lo, hi, shape, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device=g.device)


def _pow2s(lo, hi, shape, g):
    return torch.ldexp(torch.ones(shape, dtype=torch.float32, device=g.device), _ints(lo, hi, shape, g))


def _sliced(vals, dtype, fill):
    """vals [R, C] as the column slice [:, PAD/2 : PAD/2 + C] of a wider buffer whose other columns hold `fill`: a read
    outside the slice changes the result."""
    R, C = vals.shape
    buf = torch.full((R, C + PAD), fill, dtype=torch.float32, device=vals.device).to(dtype)
    buf[:, PAD // 2: PAD // 2 + C] = vals.to(dtype)
    return buf[:, PAD // 2: PAD // 2 + C]


def _bf16_operand(R, K, g, exps=(-2, 2), zeros=True):
    """{0, +-1} (or +-1) x 2^e per row, as bf16 (exact)."""
    v = _ints(-1, 1, (R, K), g) if zeros else 2 * _ints(0, 1, (R, K), g) - 1
    return (v.float() * _pow2s(exps[0], exps[1], (R, 1), g)).to(torch.bfloat16)


def _quarters(shape, g):
    """bf16 multiples of 2^-2 with magnitude <= 64."""
    return (_ints(-256, 256, shape, g).float() / 4).to(torch.bfloat16)


def _kb_exponents(M, KB, g, lo=-3, hi=3):
    """Per-(row, k-block) exponents in [lo, hi] with neighbouring k-blocks always different, so a shifted, swapped or
    repeated k-block scale changes every partial it touches."""
    span = hi - lo + 1
    steps = _ints(1, span - 1, (M, KB), g)
    steps[:, 0] = _ints(0, span - 1, (M,), g)
    return steps.cumsum(1) % span + lo


class ExactCase:
    """One call with exact operands.  `expected` is the fp64 value before the kernel's one rounding; `run(impl)` calls
    the entry point `fn` of a binding or stand-in module (or any object with that attribute)."""

    def __init__(self, fn, name, M, N, K, epilogue, **ops):
        self.fn, self.name, self.M, self.N, self.K, self.epilogue = fn, name, M, N, K, epilogue
        for k in ("a", "w", "u", "b", "col_scale", "a8", "a_scale", "w8", "w_scale", "bias", "residual", "gate",
                  "mod_index", "out", "out_scale", "block_n"):
            setattr(self, k, ops.get(k))
        self.group_rows = ops.get("group_rows", 0)
        check_budget(self)
        self.expected = reference(self)

    def kwargs(self):
        kw = dict(epilogue=self.epilogue, residual=self.residual, gate=self.gate, group_rows=self.group_rows,
                  mod_index=self.mod_index, out=self.out, block_n=self.block_n or 0)
        if self.fn == "gemm_lora" and self.col_scale is not None:
            kw["col_scale"] = self.col_scale
        if self.fn == "gemm_fp8_blocks":
            kw["out_scale"] = self.out_scale
        return kw

    def args(self):
        if self.fn == "gemm":
            return (self.a, self.w, self.bias)
        if self.fn == "gemm_lora":
            return (self.a, self.w, self.bias, self.u, self.b)
        return (self.a8, self.a_scale, self.w8, self.w_scale, self.bias)

    def run(self, impl):
        fn = impl if callable(impl) else getattr(impl, self.fn)
        return fn(*self.args(), **self.kwargs())

    def __repr__(self):
        return self.name


def _epilogue_ops(M, N, epilogue, gate_mode, g, gelu):
    """bias, residual, gate, group_rows, mod_index for one case.  gate_mode: None, "groups", "mod_index" or "alias"
    (gate with row groups, and `out` aliasing `residual`)."""
    ops = {}
    ops["bias"] = torch.full((N,), GELU_BIAS, dtype=torch.bfloat16, device=g.device) if gelu else _quarters((N,), g)
    if epilogue == EPI_BIAS_GATE_RES:
        ops["residual"] = _sliced(_quarters((M, N), g), torch.bfloat16, 0.0)
        gr = max(1, (M + 2) // 3)
        groups = -(-M // gr)
        G = groups + 2 if gate_mode == "mod_index" else groups
        gate = _pow2s(-1, 1, (G, N), g) * (2 * _ints(0, 1, (G, N), g) - 1).float()
        buf = torch.zeros(G, 2, N, dtype=torch.float32, device=g.device)   # a [G, N] view with row stride 2 N
        buf[:, 1] = gate
        ops["gate"], ops["group_rows"] = buf[:, 1], gr
        if gate_mode == "mod_index":
            ops["mod_index"] = _ints(0, G - 1, (groups,), g).to(torch.int32)
        if gate_mode == "alias":
            ops["out"] = ops["residual"]
    return ops


def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def _name(fn, M, N, K, epilogue, extra):
    return f"{fn} M={M} N={N} K={K} {EPI_NAMES[epilogue]}" + "".join(f" {k}={v}" for k, v in extra.items() if v)


def gemm_case(M, N, K, epilogue=EPI_BIAS, *, gate_mode=None, block_n=0, seed=0, device="cpu"):
    """`gemm` (bf16 operands).  For EPI_BIAS_GELU_TANH: unit-magnitude +-1 operands and bias 4096 (needs K <= 3072)."""
    g = _gen(seed, device)
    gelu = epilogue == EPI_BIAS_GELU_TANH
    exps = (0, 0) if gelu else (-2, 2)
    a = _sliced(_bf16_operand(M, K, g, exps, zeros=not gelu), torch.bfloat16, 2.0 ** 10)
    w = _bf16_operand(N, K, g, exps, zeros=not gelu)
    ops = _epilogue_ops(M, N, epilogue, gate_mode, g, gelu)
    return ExactCase("gemm", _name("gemm", M, N, K, epilogue, dict(gate=gate_mode, block_n=block_n)), M, N, K, epilogue,
                     a=a, w=w, block_n=block_n, **ops)


def lora_case(M, N, K, r, epilogue=EPI_BIAS, *, col_scale=False, gate_mode=None, block_n=0, seed=0, device="cpu"):
    """`gemm_lora`, with DoRA's col_scale (powers of two in [2^-1, 2^2]) when `col_scale`."""
    g = _gen(seed, device)
    a = _sliced(_bf16_operand(M, K, g), torch.bfloat16, 2.0 ** 10)
    w = _bf16_operand(N, K, g)
    u = _sliced(_bf16_operand(M, r, g), torch.bfloat16, 2.0 ** 10)
    b = _bf16_operand(N, r, g)
    cs = _pow2s(-1, 2, (N,), g) if col_scale else None
    ops = _epilogue_ops(M, N, epilogue, gate_mode, g, False)
    name = _name("gemm_lora", M, N, K, epilogue, dict(r=r, col_scale=col_scale, gate=gate_mode, block_n=block_n))
    return ExactCase("gemm_lora", name, M, N, K, epilogue, a=a, w=w, u=u, b=b, col_scale=cs, block_n=block_n, **ops)


def _fp8_operands(M, N, K, g, gelu, w_exps):
    if gelu:   # +-1 codes, scales in {1/2, 1}: |a . w| <= K keeps v = 4096 + a . w in the GELU regime
        a = 2 * _ints(0, 1, (M, K), g) - 1
        w = 2 * _ints(0, 1, (N, K), g) - 1
    else:
        a = _ints(-1, 1, (M, K), g)
        w = _ints(-2, 2, (N, K), g)
    a8 = _sliced(a.float(), E4M3, 448.0)
    return a8, w.float().to(E4M3), _pow2s(*w_exps, (N,), g)


def fp8_case(M, N, K, epilogue=EPI_BIAS, *, gate_mode=None, block_n=0, seed=0, device="cpu"):
    """`gemm_fp8`: per-row A scales."""
    g = _gen(seed, device)
    a8, w8, sw = _fp8_operands(M, N, K, g, False, (-3, 2))   # a_scale w_scale <= 2^5: room for gate 2 + residual
    sa = _pow2s(-3, 3, (M,), g)
    ops = _epilogue_ops(M, N, epilogue, gate_mode, g, False)
    return ExactCase("gemm_fp8", _name("gemm_fp8", M, N, K, epilogue, dict(gate=gate_mode, block_n=block_n)), M, N, K,
                     epilogue, a8=a8, a_scale=sa, w8=w8, w_scale=sw, block_n=block_n, **ops)


def fp8_blocks_case(M, N, K, epilogue=EPI_BIAS, *, a_blocks=True, gate_mode=None, block_n=0, seed=0, device="cpu"):
    """`gemm_fp8_blocks`: a_scale per (row, k-block) as a column view of a wider buffer (row stride > K / 128), or per
    row (`a_blocks=False`).  EPI_BIAS_GELU_TANH_FP8 writes into column slices of wider e4m3 / fp32 buffers filled with
    sentinels; the case keeps the buffers (`out_buf`, `scale_buf`) so a test can check the bytes outside the slices."""
    g = _gen(seed, device)
    gelu = epilogue == EPI_BIAS_GELU_TANH_FP8
    KB = K // 128
    # w_scale <= 2^2 (2^0 beyond K = 4608) keeps the scaled k-block sum plus bias, gate and residual in the fp32 budget
    a8, w8, sw = _fp8_operands(M, N, K, g, gelu, (-1, 0) if gelu else ((-3, 0) if K > 4608 else (-3, 2)))
    lo, hi = (-1, 0) if gelu else (-3, 3)
    if a_blocks:
        buf = torch.full((M, KB + 3), 2.0 ** 3, dtype=torch.float32, device=device)
        buf[:, 1:1 + KB] = torch.ldexp(torch.ones(M, KB, device=device), _kb_exponents(M, KB, g, lo, hi))
        sa = buf[:, 1:1 + KB]
    else:
        sa = _pow2s(lo, hi, (M,), g)
    ops = _epilogue_ops(M, N, epilogue, gate_mode, g, gelu)
    extra = {}
    if gelu:
        out_buf = torch.full((M, N + 2 * 128), 0x5A, dtype=torch.uint8, device=device)
        scale_buf = torch.full((M, N // 128 + 3), -7.0, dtype=torch.float32, device=device)
        ops["out"], ops["out_scale"] = out_buf[:, 128:128 + N].view(E4M3), scale_buf[:, 1:1 + N // 128]
        extra = dict(out_buf=out_buf, scale_buf=scale_buf)
    name = _name("gemm_fp8_blocks", M, N, K, epilogue, dict(a_scale="blocks" if a_blocks else "rows", gate=gate_mode,
                                                            block_n=block_n))
    case = ExactCase("gemm_fp8_blocks", name, M, N, K, epilogue, a8=a8, a_scale=sa, w8=w8, w_scale=sw,
                     block_n=block_n, **ops)
    for k, v in extra.items():
        setattr(case, k, v)
    return case


# ---- the case matrix --------------------------------------------------------------------------------------------------
# (M, N, K, block_n): every M tail (1 row, one short of / exactly / one over a 64-row half tile, 333, and 16384 rows =
# more tiles than fit on the GPU at once), ragged column tiles (N = 8 .. 520), 1 to 36 k-blocks (K = 4608 wraps the
# shared-memory stage ring many times).
FP8_GEOMS = [(1, 8, 128, 64), (63, 56, 256, 64), (64, 64, 1152, 128), (65, 72, 128, 128), (129, 136, 4608, 64),
             (333, 520, 1152, 128), (333, 520, 4608, 64), (16384, 520, 1152, 128), (129, 8, 256, 128),
             (65, 520, 256, 64)]
BLOCK_K_GEOMS = [(129, 520, 15360, 128), (333, 136, 15360, 64)]     # 120 k-blocks of per-(row, k-block) scales
FP8_GELU_GEOMS = [(1, 128, 128), (65, 384, 1152), (333, 256, 3072)]
# bf16 controls: the FP8 geometries with every tile width, plus K = 8 and 72 (a partial last k-block, zero-filled by TMA)
BF16_GEOMS = ([(M, N, K, (64, 128, 192, 256)[i % 4]) for i, (M, N, K, _) in enumerate(FP8_GEOMS)]
              + [(65, 72, 8, 128), (333, 520, 72, 256), (129, 136, 72, 64), (1, 56, 8, 192)])
LORA_GEOMS = [(1, 8, 72, 8, 64), (65, 72, 256, 8, 128), (129, 136, 128, 136, 192), (333, 520, 1152, 72, 256),
              (16384, 520, 1152, 72, 128), (63, 520, 4608, 136, 0)]
EPILOGUES = [(EPI_BIAS, None), (EPI_BIAS_GATE_RES, "groups"), (EPI_BIAS_GATE_RES, "mod_index"),
             (EPI_BIAS_GATE_RES, "alias")]


def matrix(max_m=None):
    """[(id, builder, args, kwargs)] of the bit-exact GEMM cases; `max_m` caps M (the CPU stand-in run)."""
    cap = (lambda m: m) if max_m is None else (lambda m: min(m, max_m))   # noqa: E731
    out = []

    def add(builder, *args, **kw):
        args = (cap(args[0]),) + args[1:]
        out.append((_case_id(builder, args, kw), builder, args, kw))

    for M, N, K, bn in FP8_GEOMS:
        for epi, gm in EPILOGUES:
            add(fp8_case, M, N, K, epi, gate_mode=gm, block_n=bn)
    for M, N, K, bn in FP8_GEOMS + BLOCK_K_GEOMS:
        for epi, gm in EPILOGUES:
            add(fp8_blocks_case, M, N, K, epi, gate_mode=gm, block_n=bn)
        add(fp8_blocks_case, M, N, K, EPI_BIAS, a_blocks=False, block_n=bn)
    for M, N, K in FP8_GELU_GEOMS:
        for a_blocks in (True, False):
            add(fp8_blocks_case, M, N, K, EPI_BIAS_GELU_TANH_FP8, a_blocks=a_blocks)
    for M, N, K, bn in BF16_GEOMS:
        for epi, gm in EPILOGUES + ([(EPI_BIAS_GELU_TANH, None)] if K <= 3072 else []):
            add(gemm_case, M, N, K, epi, gate_mode=gm, block_n=bn)
    for M, N, K, r, bn in LORA_GEOMS:
        for cs in (False, True):
            for epi, gm in ((EPI_BIAS, None), (EPI_BIAS_GATE_RES, "mod_index")):
                add(lora_case, M, N, K, r, epi, col_scale=cs, gate_mode=gm, block_n=bn)
    return out


def _case_id(builder, args, kw):
    return builder.__name__[:-5] + "-" + "-".join(str(x) for x in args) + "".join(
        f"-{k}={v}" for k, v in kw.items() if v is not None and not (type(v) is int and v == 0))


# ---- quantizer edges --------------------------------------------------------------------------------------------------
TIES = [1.0625, 1.1875, 2.0 ** -10, 3 * 2.0 ** -10, 5 * 2.0 ** -10, 448.0, -0.0]


def quant_edge_rows(K=256):
    """bf16 [5, K] rows: (0) the tie table (and its negatives) with amax 448, s = 1, in every 128-column block; (1) all -0;
    (2) an all-zero first block before a block of ties; (3) the ties scaled by 2^-4 with amax 28, s = 2^-4; (4) amax 300,
    s = 300 / 448, not a power of two."""
    t = torch.tensor(TIES + [-v for v in TIES[:-1]], dtype=torch.float32)
    x = torch.zeros(5, K)
    for b in range(K // 128):
        x[0, 128 * b: 128 * b + len(t)] = t
        x[3, 128 * b: 128 * b + len(t)] = t * 2.0 ** -4
        x[3, 128 * b + len(t)] = 28.0
    x[1] = -0.0
    x[2, 128: 128 + len(t)] = t
    x[4] = torch.linspace(-300, 300, K)
    x[4, :64] = torch.tensor([1.0625, 1.1875, 9.0, 13.0, 2.0 ** -8, 40.0, 104.0, 208.0]).repeat(8) * (300.0 / 448.0)
    return x.to(torch.bfloat16)


def quant_expected(x, block):
    """torch's fp32 x / s cast to e4m3, s = amax / 448 per `block` columns (1 for a zero block)."""
    R, K = x.shape
    xb = x.float().view(R, K // block, block)
    amax = xb.abs().amax(-1)
    s = torch.where(amax > 0, amax / torch.full_like(amax, 448.0), torch.ones_like(amax))   # IEEE quotient
    return (xb / s[..., None]).clamp(-448.0, 448.0).to(E4M3).view(R, K), s


# ---- comparison -------------------------------------------------------------------------------------------------------
_INT_VIEW = {torch.bfloat16: torch.int16, torch.float32: torch.int32, E4M3: torch.uint8}


def first_mismatch(got, want, *, signed_zero=False):
    """None when got and want hold identical bit patterns (-0 == +0 unless `signed_zero`), else a description of how
    many elements differ and the first differing (row, column) with both values."""
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    it = _INT_VIEW[got.dtype]
    gb, wb = got.contiguous().view(it), want.contiguous().view(it)
    bad = gb != wb
    if not signed_zero:
        bad &= ~((got.float() == 0) & (want.float() == 0))
    if not bool(bad.any()):
        return None
    idx = tuple(int(i) for i in bad.nonzero()[0])
    mask = 0xFF if it == torch.uint8 else (1 << (8 * got.element_size())) - 1
    return (f"{int(bad.sum())} of {bad.numel()} elements differ; first at (row, column) {idx}: "
            f"got {float(got[idx].float()):.9g} (0x{int(gb[idx]) & mask:0{2 * got.element_size()}x}), "
            f"want {float(want[idx].float()):.9g} (0x{int(wb[idx]) & mask:0{2 * got.element_size()}x})")


def assert_bits(what, got, want, **kw):
    msg = first_mismatch(got, want, **kw)
    assert msg is None, f"{what}: {msg}"


def conv_box(t_out, h_out, w_out):
    """(Tt, Ht, Wt) of the CTA box osb_conv3d_ndhwc picks: least padded work, wide W first."""
    best, box = 1e30, None
    for wl in range(7, 2, -1):
        for hl in range(0, 8 - wl):
            Wt, Ht, Tt = 1 << wl, 1 << hl, 128 >> (wl + hl)
            work = (-(-w_out // Wt) * Wt) * (-(-h_out // Ht) * Ht) * (-(-t_out // Tt) * Tt)
            if work < best * 0.999:
                best, box = work, (Tt, Ht, Wt)
    return box
