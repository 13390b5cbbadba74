"""GPU parity of each C-ABI kernel against a plain PyTorch fp32 restatement of the same op on
identical bf16-rounded inputs.  Tolerance: the kernels accumulate in fp32 and round ONCE to bf16,
so rel-L2 vs the fp32 result must stay within one bf16 rounding (2e-3); attention additionally
rounds P to bf16 before PV (as flash-attention does), bounded at 4e-3."""
import math

import pytest
import torch

from tests.util import BF16_ONE_ROUNDING_REL_L2, report

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def osb():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import osb200

    osb200.init(0)
    return osb200


def _randn(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,C,group_rows", [(1000, 1152, 250), (77, 3072, 77), (4096, 384, 1024), (9, 64, 3),
                                                (4099, 1152, 4099), (16384, 1152, 8192)])
def test_ln_modulate(osb, rows, C, group_rows):
    x = _randn(rows, C, seed=1) * 3 + 0.5
    G = (rows + group_rows - 1) // group_rows
    mod = torch.randn(G, 2, C, device="cuda") * 0.5
    shift, scale = mod[:, 0], mod[:, 1]
    y = osb.ln_modulate(x, shift, scale, group_rows=group_rows)
    xf = x.float()
    ref = torch.nn.functional.layer_norm(xf, (C,), eps=1e-6)
    g = torch.arange(rows, device="cuda") // group_rows
    ref = ref * (1 + scale[g]) + shift[g]
    r, _ = report(f"ln_modulate {rows}x{C}", y, ref)
    assert r < BF16_ONE_ROUNDING_REL_L2


def test_ln_modulate_index(osb):
    rows, C, S = 512, 1152, 64
    x = _randn(rows, C, seed=2)
    mod = torch.randn(4, 2, C, device="cuda")
    idx = torch.randint(0, 4, (rows // S,), device="cuda", dtype=torch.int32)
    y = osb.ln_modulate(x, mod[:, 0], mod[:, 1], group_rows=S, mod_index=idx)
    g = idx.long()[torch.arange(rows, device="cuda") // S]
    ref = torch.nn.functional.layer_norm(x.float(), (C,), eps=1e-6) * (1 + mod[g, 1]) + mod[g, 0]
    r, _ = report("ln_modulate idx", y, ref)
    assert r < BF16_ONE_ROUNDING_REL_L2


# ------------------------------------------------------------------------------------------------
GEMM_SHAPES = [
    (128, 64, 64),      # one tile, one k-block
    (256, 256, 128),
    (300, 2304, 1152),  # ragged M (T5 tokens x kv_linear)
    (1000, 1152, 4608),
    (2048, 3456, 1152),
    (515, 72, 200),     # ragged everything: N, K not multiples of the tile
]


def _gemm(osb, *args, cta_group, **kw):
    """cta_group is accepted for ABI compatibility and selects nothing on sm_90a: any value must give the bits of the
    default."""
    out = osb.gemm(*args, cta_group=cta_group, **kw)
    if cta_group:
        assert torch.equal(out, osb.gemm(*args, cta_group=0, **kw)), f"cta_group={cta_group} changed the result"
    return out


def _attn_short(osb, q, k, v, out, **kw):
    """The implementation switch (osb_attn_short_args.reserved) selects nothing on sm_90a: any value must give the bits
    of the default (rows the call does not write are carried over by the clone)."""
    osb.attn_short(q, k, v, out, **kw)
    if kw.get("impl", 0):
        alt = out.clone()
        osb.attn_short(q, k, v, alt, **{**kw, "impl": 0})
        assert torch.equal(alt, out), f"impl={kw['impl']} changed the result"
    return out


@pytest.mark.parametrize("cta", [1, 2])
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_bias(osb, M, N, K, cta):
    a = _randn(M, K, seed=3)
    w = _randn(N, K, scale=K ** -0.5, seed=4)
    b = _randn(N, seed=5)
    out = _gemm(osb, a, w, b, cta_group=cta)
    ref = a.float() @ w.float().t() + b.float()
    r, _ = report(f"gemm bias {M}x{N}x{K} cta{cta}", out, ref)
    assert r < BF16_ONE_ROUNDING_REL_L2


@pytest.mark.parametrize("cta", [1, 2])
@pytest.mark.parametrize("bn", [64, 128, 192, 256])
def test_gemm_block_n(osb, bn, cta):
    M, N, K = 777, 1152, 1152
    a = _randn(M, K, seed=6)
    w = _randn(N, K, scale=K ** -0.5, seed=7)
    out = _gemm(osb, a, w, None, cta_group=cta, block_n=bn)
    ref = a.float() @ w.float().t()
    r, _ = report(f"gemm bn{bn} cta{cta}", out, ref)
    assert r < BF16_ONE_ROUNDING_REL_L2


@pytest.mark.parametrize("cta", [1, 2])
def test_gemm_gelu(osb, cta):
    M, N, K = 1024, 4608, 1152
    a = _randn(M, K, seed=8)
    w = _randn(N, K, scale=K ** -0.5, seed=9)
    b = _randn(N, seed=10)
    out = _gemm(osb, a, w, b, epilogue=osb.EPI_BIAS_GELU_TANH, cta_group=cta)
    ref = torch.nn.functional.gelu(a.float() @ w.float().t() + b.float(), approximate="tanh")
    r, _ = report(f"gemm gelu cta{cta}", out, ref)
    assert r < BF16_ONE_ROUNDING_REL_L2


@pytest.mark.parametrize("cta", [1, 2])
@pytest.mark.parametrize("use_gate", [True, False])
def test_gemm_gate_residual(osb, cta, use_gate):
    M, N, K, group = 1536, 1152, 4608, 512
    a = _randn(M, K, seed=11)
    w = _randn(N, K, scale=K ** -0.5, seed=12)
    b = _randn(N, seed=13)
    res = _randn(M, N, seed=14)
    gate = torch.randn(M // group, N, device="cuda") if use_gate else None
    out = _gemm(osb, a, w, b, epilogue=osb.EPI_BIAS_GATE_RES, residual=res, gate=gate, group_rows=group, cta_group=cta)
    lin = a.float() @ w.float().t() + b.float()
    if use_gate:
        lin = lin * gate[torch.arange(M, device="cuda") // group]
    ref = res.float() + lin
    r, _ = report(f"gemm gate_res cta{cta} gate={use_gate}", out, ref)
    assert r < BF16_ONE_ROUNDING_REL_L2


def test_gemm_inplace_residual_and_strided_a(osb):
    # x = x + gate * proj(attn) written in place; A is a column slice of a wider buffer
    M, N, K = 640, 1152, 1152
    wide = _randn(M, 2 * K, seed=15)
    a = wide[:, K:]
    w = _randn(N, K, scale=K ** -0.5, seed=16)
    x = _randn(M, N, seed=17)
    x0 = x.clone()
    gate = torch.randn(1, N, device="cuda")
    osb.gemm(a, w, None, epilogue=osb.EPI_BIAS_GATE_RES, residual=x, gate=gate, group_rows=M, out=x)
    ref = x0.float() + gate * (a.float() @ w.float().t())
    r, _ = report("gemm inplace", x, ref)
    assert r < BF16_ONE_ROUNDING_REL_L2


def test_gemm_large_persistent(osb):
    # many k-blocks per tile: exercises the smem ring wrap and both mbarrier phases
    M, N, K = 16384, 1152, 1152
    a = _randn(M, K, seed=18)
    w = _randn(N, K, scale=K ** -0.5, seed=19)
    b = _randn(N, seed=20)
    ref = a.float() @ w.float().t() + b.float()
    for cta in (1, 2):
        out = _gemm(osb, a, w, b, cta_group=cta)
        r, _ = report(f"gemm large cta{cta}", out, ref)
        assert r < BF16_ONE_ROUNDING_REL_L2


# ------------------------------------------------------------------------------------------------
def _attn_ref(q, k, v, qw, kw, cos, sin, scale, kv_len=None):
    """q,k,v: fp32 [n, H, L, D]; returns [n, H, Lq, D] (fp32 math, oracle restatement)."""
    def rms(x, w):
        return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w

    def rope(x, cos, sin):
        L = x.shape[-2]
        x1, x2 = x[..., 0::2], x[..., 1::2]
        c, s = cos[:L], sin[:L]
        o = torch.stack((x1 * c - x2 * s, x2 * c + x1 * s), dim=-1)
        return o.flatten(-2)

    if qw is not None:
        q, k = rms(q, qw.float()), rms(k, kw.float())
    if cos is not None:
        q, k = rope(q, cos, sin), rope(k, cos, sin)
    s = (q @ k.transpose(-1, -2)) * scale
    if kv_len is not None:
        mask = torch.arange(k.shape[-2], device=q.device)[None, :] >= kv_len[:, None]
        s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    return torch.softmax(s, dim=-1) @ v


def _rope_tables(L, D):
    inv = 1.0 / (10000 ** (torch.arange(0, D, 2, device="cuda").float() / D))
    ang = torch.arange(L, device="cuda").float()[:, None] * inv[None]
    return ang.cos().contiguous(), ang.sin().contiguous()


IMPLS = [1, 2, 3, 4]  # values of the implementation switch (osb_attn_short_args.reserved): see _attn_short


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("D,H", [(72, 4), (64, 3), (128, 2)])
@pytest.mark.parametrize("mode", ["spatial", "temporal"])
def test_attn_self(osb, D, H, mode, impl):
    B, T, S = 2, 16, 256
    if mode == "temporal":
        T, S = 64, 24
    C = H * D
    N = T * S
    qkv = _randn(B * N, 3 * C, seed=21)
    qw, kw = _randn(D, seed=22) * 0.2 + 1, _randn(D, seed=23) * 0.2 + 1
    use_rope = mode == "temporal"
    cos, sin = _rope_tables(T, D) if use_rope else (None, None)
    out = torch.zeros(B * N, C, dtype=torch.bfloat16, device="cuda")
    q2, k2, v2 = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    if mode == "spatial":
        strides = (N, S, 1)
        _attn_short(osb, q2, k2, v2, out, num_seqs=B * T, seqs_per_batch=T, q_strides=strides, k_strides=strides,
                       Lq=S, Lk=S, num_heads=H, head_dim=D, q_norm_w=qw, k_norm_w=kw, impl=impl)
        x = qkv.float().view(B * T, S, 3, H, D).permute(2, 0, 3, 1, 4)
        ref = _attn_ref(x[0], x[1], x[2], qw, kw, None, None, D ** -0.5)       # [B*T, H, S, D]
        ref = ref.permute(0, 2, 1, 3).reshape(B * N, C)
    else:
        strides = (N, 1, S)
        _attn_short(osb, q2, k2, v2, out, num_seqs=B * S, seqs_per_batch=S, q_strides=strides, k_strides=strides,
                       Lq=T, Lk=T, num_heads=H, head_dim=D, q_norm_w=qw, k_norm_w=kw, rope_cos=cos, rope_sin=sin, impl=impl)
        x = qkv.float().view(B, T, S, 3, H, D).permute(3, 0, 2, 4, 1, 5).reshape(3, B * S, H, T, D)
        ref = _attn_ref(x[0], x[1], x[2], qw, kw, cos, sin, D ** -0.5)          # [B*S, H, T, D]
        ref = ref.view(B, S, H, T, D).permute(0, 3, 1, 2, 4).reshape(B * N, C)
    r, _ = report(f"attn {mode} D{D} impl{impl}", out, ref)
    assert r < 4e-3


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("Ly", [300, 77])
def test_attn_cross(osb, Ly, impl):
    B, N, H, D = 2, 640, 4, 72
    C = H * D
    q = _randn(B * N, C, seed=24)
    kv = _randn(B * Ly, 2 * C, seed=25)
    lens = torch.tensor([Ly, max(1, Ly // 3)], device="cuda", dtype=torch.int32)
    out = torch.zeros(B * N, C, dtype=torch.bfloat16, device="cuda")
    _attn_short(osb, q, kv[:, :C], kv[:, C:], out, num_seqs=B, seqs_per_batch=1, q_strides=(N, 0, 1),
                   k_strides=(Ly, 0, 1), Lq=N, Lk=Ly, num_heads=H, head_dim=D, kv_lens=lens, impl=impl)
    qf = q.float().view(B, N, H, D).permute(0, 2, 1, 3)
    kvf = kv.float().view(B, Ly, 2, H, D).permute(2, 0, 3, 1, 4)
    ref = _attn_ref(qf, kvf[0], kvf[1], None, None, None, None, D ** -0.5, kv_len=lens)
    ref = ref.permute(0, 2, 1, 3).reshape(B * N, C)
    r, _ = report(f"attn cross Ly{Ly} impl{impl}", out, ref)
    assert r < 4e-3


@pytest.mark.parametrize("impl", [1, 3, 4])
@pytest.mark.parametrize("T,S", [(4, 24), (3, 40), (5, 7)])
def test_attn_packed_ragged(osb, T, S, impl):
    """Short sequences packed G per 128-row tile where G*L < 128 and rows of one warp belong to different sequences
    (XS parity shapes: S=24 -> G=5): block-diagonal masking must not make warp-collective loads or shuffles diverge."""
    B, H, D = 2, 4, 72
    C, N = H * D, T * S
    qkv = _randn(B * N, 3 * C, seed=41)
    qw, kw = _randn(D, seed=42) * 0.2 + 1, _randn(D, seed=43) * 0.2 + 1
    q2, k2, v2 = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    for mode in ("spatial", "temporal"):
        out = torch.zeros(B * N, C, dtype=torch.bfloat16, device="cuda")
        if mode == "spatial":
            st = (N, S, 1)
            _attn_short(osb, q2, k2, v2, out, num_seqs=B * T, seqs_per_batch=T, q_strides=st, k_strides=st, Lq=S, Lk=S,
                           num_heads=H, head_dim=D, q_norm_w=qw, k_norm_w=kw, impl=impl)
            x = qkv.float().view(B * T, S, 3, H, D).permute(2, 0, 3, 1, 4)
            ref = _attn_ref(x[0], x[1], x[2], qw, kw, None, None, D ** -0.5).permute(0, 2, 1, 3).reshape(B * N, C)
        else:
            cos, sin = _rope_tables(T, D)
            st = (N, 1, S)
            _attn_short(osb, q2, k2, v2, out, num_seqs=B * S, seqs_per_batch=S, q_strides=st, k_strides=st, Lq=T, Lk=T,
                           num_heads=H, head_dim=D, q_norm_w=qw, k_norm_w=kw, rope_cos=cos, rope_sin=sin, impl=impl)
            x = qkv.float().view(B, T, S, 3, H, D).permute(3, 0, 2, 4, 1, 5).reshape(3, B * S, H, T, D)
            ref = _attn_ref(x[0], x[1], x[2], qw, kw, cos, sin, D ** -0.5)
            ref = ref.view(B, S, H, T, D).permute(0, 3, 1, 2, 4).reshape(B * N, C)
        r, _ = report(f"attn packed ragged {mode} T{T} S{S} impl{impl}", out, ref)
        assert r < 4e-3


@pytest.mark.parametrize("big_logits", [False, True])
@pytest.mark.parametrize("mode", ["spatial", "temporal", "cross"])
def test_attn_pingpong_many_sets(osb, mode, big_logits):
    """The two-slot kernel when every CTA walks several key sets: ring reuse of the K/V stages, jobs of one set split
    between CTAs (cross: 41 q-tiles per head over 148 CTAs), odd job counts.  big_logits scales q / the norm weights so
    that the Cauchy-Schwarz logit bound exceeds the one-pass limit and the two-pass (online max) path runs."""
    H, D = 4, 72
    C = H * D
    amp = 6.0 if big_logits else 1.0   # bound ~ 12 * amp log2-units; the one-pass limit is 60
    if mode == "cross":
        B, N, Ly = 2, 128 * 41 - 50, 300
        q = _randn(B * N, C, seed=31) * amp
        kv = _randn(B * Ly, 2 * C, seed=32)
        lens = torch.tensor([260, 300], device="cuda", dtype=torch.int32)
        out = torch.zeros(B * N, C, dtype=torch.bfloat16, device="cuda")
        _attn_short(osb, q, kv[:, :C], kv[:, C:], out, num_seqs=B, seqs_per_batch=1, q_strides=(N, 0, 1),
                       k_strides=(Ly, 0, 1), Lq=N, Lk=Ly, num_heads=H, head_dim=D, kv_lens=lens, impl=4)
        qf = q.float().view(B, N, H, D).permute(0, 2, 1, 3)
        kvf = kv.float().view(B, Ly, 2, H, D).permute(2, 0, 3, 1, 4)
        ref = _attn_ref(qf, kvf[0], kvf[1], None, None, None, None, D ** -0.5, kv_len=lens).permute(0, 2, 1, 3).reshape(B * N, C)
    else:
        B, T, S = (1, 331, 256) if mode == "spatial" else (1, 64, 1307)
        N = T * S
        qkv = _randn(B * N, 3 * C, seed=33)
        qw, kw = (_randn(D, seed=34) * 0.2 + 1) * amp, _randn(D, seed=35) * 0.2 + 1
        out = torch.zeros(B * N, C, dtype=torch.bfloat16, device="cuda")
        q2, k2, v2 = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        if mode == "spatial":
            st = (N, S, 1)
            _attn_short(osb, q2, k2, v2, out, num_seqs=B * T, seqs_per_batch=T, q_strides=st, k_strides=st, Lq=S, Lk=S,
                           num_heads=H, head_dim=D, q_norm_w=qw, k_norm_w=kw, impl=4)
            x = qkv.float().view(B * T, S, 3, H, D).permute(2, 0, 3, 1, 4)
            ref = _attn_ref(x[0], x[1], x[2], qw, kw, None, None, D ** -0.5).permute(0, 2, 1, 3).reshape(B * N, C)
        else:
            cos, sin = _rope_tables(T, D)
            st = (N, 1, S)
            _attn_short(osb, q2, k2, v2, out, num_seqs=B * S, seqs_per_batch=S, q_strides=st, k_strides=st, Lq=T, Lk=T,
                           num_heads=H, head_dim=D, q_norm_w=qw, k_norm_w=kw, rope_cos=cos, rope_sin=sin, impl=4)
            x = qkv.float().view(B, T, S, 3, H, D).permute(3, 0, 2, 4, 1, 5).reshape(3, B * S, H, T, D)
            ref = _attn_ref(x[0], x[1], x[2], qw, kw, cos, sin, D ** -0.5)
            ref = ref.view(B, S, H, T, D).permute(0, 3, 1, 2, 4).reshape(B * N, C)
    r, _ = report(f"attn ping-pong many sets {mode} big_logits={big_logits}", out, ref)
    assert r < (2e-2 if big_logits else 4e-3)   # large logits amplify the bf16 rounding of q-hat / k-hat themselves


@pytest.mark.parametrize("impl", [2, 3])
@pytest.mark.parametrize("D", [72, 128])
def test_attn_long_sequence(osb, D, impl):
    """Streaming path: many key blocks per query tile (online softmax + O rescaling), L not a multiple of anything."""
    H, nseq, L = 2, 2, 1000
    C = H * D
    qkv = _randn(nseq * L, 3 * C, seed=31)
    qw, kw = _randn(D, seed=32) * 0.2 + 1, _randn(D, seed=33) * 0.2 + 1
    qw2, kw2 = _randn(D, seed=34) * 0.2 + 1, _randn(D, seed=35) * 0.2 + 1
    cos, sin = _rope_tables(L, D)
    out = torch.zeros(nseq * L, C, dtype=torch.bfloat16, device="cuda")
    split = 100
    _attn_short(osb, qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, num_seqs=nseq, seqs_per_batch=1, q_strides=(L, 0, 1),
                   k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H, head_dim=D, q_norm_w=qw, k_norm_w=kw, q_norm_w2=qw2,
                   k_norm_w2=kw2, norm_split=split, rope_cos=cos, rope_sin=sin, impl=impl)
    x = qkv.float().view(nseq, L, 3, H, D).permute(2, 0, 3, 1, 4)

    def rms(t, w1, w2):
        n = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6)
        w = torch.where((torch.arange(L, device="cuda") >= split)[:, None], w2.float()[None], w1.float()[None])
        return n * w

    ref = _attn_ref(rms(x[0], qw, qw2), rms(x[1], kw, kw2), x[2], None, None, cos, sin, D ** -0.5)
    ref = ref.permute(0, 2, 1, 3).reshape(nseq * L, C)
    r, _ = report(f"attn long L{L} D{D} impl{impl}", out, ref)
    assert r < 4e-3


def test_attn_ragged_tail(osb):
    # Lq not a multiple of 128 and an odd number of packed sequences: exercises masking of rows/slots
    D, H = 72, 2
    C = H * D
    for (nseq, L) in [(5, 48), (3, 200)]:
        qkv = _randn(nseq * L, 3 * C, seed=26)
        out = torch.zeros(nseq * L, C, dtype=torch.bfloat16, device="cuda")
        _attn_short(osb, qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, num_seqs=nseq, seqs_per_batch=nseq,
                       q_strides=(0, L, 1), k_strides=(0, L, 1), Lq=L, Lk=L, num_heads=H, head_dim=D)
        x = qkv.float().view(nseq, L, 3, H, D).permute(2, 0, 3, 1, 4)
        ref = _attn_ref(x[0], x[1], x[2], None, None, None, None, D ** -0.5).permute(0, 2, 1, 3).reshape(nseq * L, C)
        r, _ = report(f"attn ragged {nseq}x{L}", out, ref)
        assert r < 4e-3


def test_errors_are_loud(osb):
    a = _randn(64, 60, seed=1)  # K not a multiple of 8
    w = _randn(64, 60, seed=2)
    with pytest.raises(osb.OsbError):
        osb.gemm(a, w)
    with pytest.raises(osb.OsbError):
        osb.gemm(a.cpu(), w.cpu())
