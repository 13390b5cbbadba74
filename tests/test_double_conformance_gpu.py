"""Conformance of the CPU double of the binding (tests/fake_osb200.py) with the osb200 kernels, element by element.

Most host-side evidence of this project runs on the CPU against the double, so the double is itself a reference: this
module pins it to the kernels.  Every case builds its inputs on the CPU, runs the double there (ACC_DTYPE = fp32, as the
host tests use it) and the binding on the GPU with the same bf16 bits, and compares EVERY element against a bound
derived from the operation's arithmetic (never a tuned tolerance).  `_check` prints one line per case: the largest
|delta| / bound and the fraction of bit-identical elements.

Bound classes
  exact        copies, index arithmetic and zero fill: bit-identical.
  one rounding the op is fp32 arithmetic rounded once to bf16 on both sides:
                   |k - d| <= ulp_bf16(max(|k|, |d|)) + E
               The ulp term covers the two final roundings (half an ulp each).  E bounds the distance between the two
               fp32 results: Higham's a-priori bound gamma_n * M per side, M the op's magnitude (the same expression
               on absolute values, in fp64), scaled through the epilogue and with the documented error of the
               approximate device functions added.  It holds for every summation order, so it cannot flake.
  attention    see _attn_eps.
"""
import itertools
import math

import pytest
import torch
import torch.nn.functional as TF

from tests import fake_osb200 as F_
from tests.models import mmdit_ids, mmdit_model, stdit3_inputs, stdit3_pair, tiny_vae
from tests.sampling_toys import toy_model
from tests.util import load_golden, read_tiles

pytestmark = pytest.mark.gpu

U = 2.0 ** -24      # fp32 unit roundoff (round to nearest): the double's CPU arithmetic and the CUDA-core epilogues
U_TC = 2.0 ** -23   # tensor-core accumulation: its rounding mode is not documented, so charge a whole fp32 ulp per add


def gam(n, u=U):
    """Higham's gamma_n = n u / (1 - n u): relative error bound of n successive fp32 roundings."""
    return n * u / (1.0 - n * u)


def gam2(n):
    """Distance between a tensor-core (or CUDA-core) fp32 result and the CPU fp32 one, relative to the magnitude M."""
    return gam(n, U_TC) + gam(n, U)


def ulp_bf16(x):
    """bf16 ulp at |x|: x = m 2^e with m in [0.5, 1) has 8 significant bits, ulp 2^(e - 8); subnormal floor 2^-133."""
    _, e = torch.frexp(x.double().abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - 8).clamp_min(2.0 ** -133)


def ulp_fp32(x):
    _, e = torch.frexp(x.double().abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - 24).clamp_min(2.0 ** -149)


def _check(name, got, want, err=None, ulp=ulp_bf16, verbose=True):
    """got: kernel result, want: the double's.  err None: bit-identical required; else |got - want| <= ulp(max) + err."""
    k, d = got.detach().cpu(), want.detach().cpu()
    assert k.shape == d.shape and k.dtype == d.dtype, (name, k.shape, d.shape, k.dtype, d.dtype)
    ib = {torch.bfloat16: torch.int16, torch.float32: torch.int32}[k.dtype]
    same = k.contiguous().view(ib) == d.contiguous().view(ib)
    frac = float(same.double().mean()) if same.numel() else 1.0
    kd, dd = k.double(), d.double()
    assert torch.isfinite(kd).all() and torch.isfinite(dd).all(), f"{name}: non-finite output"
    if err is None:
        ratio = 0.0 if bool(same.all()) else math.inf
    else:
        bound = ulp(torch.maximum(kd.abs(), dd.abs())) + err.double().expand_as(kd)
        ratio = float(((kd - dd).abs() / bound).max()) if kd.numel() else 0.0
    kind = "exact" if err is None else "bound"
    if verbose:
        print(f"[conformance] {name}: {kind} max|d|/bound={ratio:.3f} bit-identical={frac:.4f} n={k.numel()}")
    assert ratio <= 1.0, f"{name}: max |delta| / bound = {ratio}"
    return ratio, int(same.sum()), same.numel()


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


def _launches(osb, real_fn, fake_fn):
    """Run both; the kernel launch count must advance by what the double counts for the same call."""
    l0, f0 = osb.launch_count(), F_.launch_count()
    r = real_fn()
    torch.cuda.synchronize()
    f = fake_fn()
    dl, df = osb.launch_count() - l0, F_.launch_count() - f0
    assert dl == df, f"launch count: kernels {dl}, double {df}"
    return r, f


def _quiet(fn):
    """Run a double entry point for a bound computation without counting it as a launch."""
    n, c = F_._launches, len(F_.calls)
    try:
        return fn()
    finally:
        F_._launches = n
        del F_.calls[c:]


# ---- error budgets E (fp64, CPU), shared by the hand-picked cases and the recorded replay ---------------------------
def _d(t):
    return None if t is None else t.detach().cpu().double()


def err_gemm(a, w, bias=None, *, epilogue=0, residual=None, gate=None, group_rows=0, mod_index=None, u=None, b=None,
             **_):
    """GEMM / LoRA GEMM.  v = sum_k a w + [sum_r u b] + bias is n = K + r + 1 fp32 adds of exact bf16 products:
    |v_k - v_d| <= gam2(n) Mv, Mv = |a| |w|^T + |u| |b|^T + |bias|.
      BIAS       E = gam2(n) Mv
      GELU(tanh) E = 1.13 gam2(n) Mv + |v| (2^-11.987 + gam(16)): GELU's slope is <= 1.13; the kernel's tanh.approx.f32
                 has relative error <= 2^-10.987 (PTX ISA) and enters as 0.5 x tanh; the polynomial, the products and
                 torch's CPU GELU are < 16 more fp32 roundings of quantities <= |x|.
      GATE_RES   v g + r: two more roundings, E = gam2(n + 2) (|g| Mv + |r|)."""
    a, w, bias, residual, gate = _d(a), _d(w), _d(bias), _d(residual), _d(gate)
    M = a.shape[0]
    mv = a.abs() @ w.abs().t()
    n = a.shape[1] + 1
    if u is not None:
        mv = mv + _d(u).abs() @ _d(b).abs().t()
        n += u.shape[1]
    if bias is not None:
        mv = mv + bias.abs()
    if epilogue == 1:
        v = a @ w.t() + (_d(u) @ _d(b).t() if u is not None else 0) + (bias if bias is not None else 0)
        return 1.13 * gam2(n) * mv + v.abs() * (2.0 ** -11.987 + gam(16))
    if epilogue == 2:
        gm = 1.0
        if gate is not None:
            g = torch.arange(M) // (group_rows if group_rows > 0 else M)
            if mod_index is not None:
                g = mod_index.cpu().long()[g]
            gm = gate.abs()[g]
        return gam2(n + 2) * (gm * mv + (residual.abs() if residual is not None else 0))
    return gam2(n) * mv


def err_ln(x, shift, scale, *, group_rows, mod_index=None, eps=1e-6, **_):
    """LayerNorm + modulate, y = (x - mu) r (1 + s) + h over a row of C elements, both sides fp32 two-pass:
      mu: C adds and a division per side          |d mu| <= E_mu = 2 gam(C + 1) mean|x|
      var = mean((x - mu')^2) = var + (mu' - mu)^2 + fp32 error gam(C + 3) (var + E_mu^2) per side
      r = (var + eps)^-1/2: relative error <= (d var) / (2 (var + eps)) + 6u (rsqrtf 2 ulp, CPU 1 ulp)
      y: |dy| <= |1 + s| r (E_mu + |x - mu| eps_r) + 2 gam(4) (|x - mu| r |1 + s| + |h|)."""
    x, shift, scale = _d(x), _d(shift), _d(scale)
    rows, C = x.shape
    g = torch.arange(rows) // (group_rows if group_rows > 0 else rows)
    if mod_index is not None:
        g = mod_index.cpu().long()[g]
    s, h = scale[g], shift[g]
    mu = x.mean(-1, keepdim=True)
    var = (x - mu).pow(2).mean(-1, keepdim=True)
    e_mu = 2 * gam(C + 1) * x.abs().mean(-1, keepdim=True)
    d_var = 2 * gam(C + 3) * (var + e_mu ** 2) + e_mu ** 2
    eps_r = d_var / (2 * (var + eps)) + 6 * U
    r = (var + eps).rsqrt()
    xc = (x - mu).abs()
    return (1 + s).abs() * r * (e_mu + xc * eps_r) + 2 * gam(4) * (xc * r * (1 + s).abs() + h.abs())


def _attn_eps(D, keys, smax):
    """Relative error budget of one attention output element, as a multiple of (P |V|)_{r,d} (P normalised).
    Both sides feed the same bf16 q-hat, k-hat and v; they differ in
      - the bf16 rounding of P: the double rounds exp(s - m_final), the kernel exp(s - m_running) (and rescales by
        alpha in fp32).  Each is within 2^-8 (relative) of the exact P, so the two are within 2^-7;
      - the scores: D exact bf16 products summed in fp32 (gam(D) S per side, S = max |q-hat| |k-hat| scale), the max
        subtracted from them and the exponent argument rounded: eps_s = 4 gam(D + 2) S + 2u S + 2^-21 for ex2.approx
        (relative error < 2^-22 on the H100) - relative error of every P entry;
      - the sums: l over `keys` unrounded P (gam(keys) per side), the PV accumulation (gam2(keys)), the online-softmax
        rescales (<= keys / 64 + 1 factors alpha, each 2^-21 + u) and the final division (u per side)."""
    eps_s = 4 * gam(D + 2) * smax + 2 * U * smax + 2.0 ** -21
    nb = keys / 64 + 1
    return 2.0 ** -7 * (1 + eps_s) + 2 * eps_s + 2 * gam(keys) + gam2(keys) + 2 * nb * (2.0 ** -21 + U) + 2 * U


# (P |V|) is taken from the double run on |v|: its output is bf16(sum bf16(P) |v| / l) >= (1 - 2^-8)^2 (P |V|) up to fp32
# noise, so (P |V|) <= 1.01 x that output.
PV_SLACK = 1.01


def _head_norm_max(x, H, D, w=None, w2=None):
    """Largest L2 norm of a staged head row: RMSNorm gives norm sqrt(D) max|w| at most, RoPE preserves pair norms, the bf16
    rounding of the staged operand adds < 2^-8 (1.01 covers both)."""
    if w is not None:
        wm = float(w.detach().abs().max())
        if w2 is not None:
            wm = max(wm, float(w2.detach().abs().max()))
        return 1.01 * math.sqrt(D) * wm
    return 1.01 * float(_d(x)[:, : H * D].reshape(-1, H, D).norm(dim=-1).max())


def err_attn_short(q, k, v, out, **kw):
    """E for osb_attn_short: eps * (P |V|), rows the call does not write get E = 0 (they must stay bit-identical)."""
    H, D = kw["num_heads"], kw["head_dim"]
    scale = kw.get("softmax_scale") or D ** -0.5
    smax = scale * _head_norm_max(q, H, D, kw.get("q_norm_w"), kw.get("q_norm_w2")) * \
        _head_norm_max(k, H, D, kw.get("k_norm_w"), kw.get("k_norm_w2"))
    G = 128 // kw["Lq"] if kw["Lq"] < 128 else 1
    pv = torch.zeros_like(out)
    _quiet(lambda: F_.attn_short(q, k, v.abs(), pv, **kw))
    return PV_SLACK * _attn_eps(D, G * kw["Lk"], smax) * pv.double()


def err_conv(x_pad, w_packed, bias, *, out_thw, stride=(1, 1, 1), taps=(3, 3, 3), narrow=False, residual=None, **_):
    """Implicit-GEMM convolution: n = kt kh kw Cp products (narrow: kt kh 64), + bias + residual:
    E = gam2(n + 2) (conv(|x|, |w|) + |bias| + |residual|)."""
    kt, kh, kw = taps
    cout = w_packed.shape[0]
    cp = x_pad.shape[-1]
    wp = _d(w_packed).abs()
    if narrow:
        w = wp.view(cout, kt * kh, 64)[:, :, : kw * cp].reshape(cout, kt, kh, kw, cp)
        n = kt * kh * 64
    else:
        w = wp.view(cout, kt, kh, kw, cp)
        n = kt * kh * kw * cp
    m = TF.conv3d(_d(x_pad).abs().permute(0, 4, 1, 2, 3), w.permute(0, 4, 1, 2, 3), stride=stride)
    m = m[:, :, : out_thw[0], : out_thw[1], : out_thw[2]].permute(0, 2, 3, 4, 1)
    if bias is not None:
        m = m + _d(bias).abs()
    if residual is not None:
        m = m + _d(residual).abs()
    return gam2(n + 2) * m


def err_vae_prep(x, *, stats=None, gamma=None, beta=None, groups=32, silu=False, up=(1, 1, 1), pad=(0, 0, 0), cp=None,
                 **_):
    """E on the unpadded, un-upsampled element (the copy / padding are exact and map E along with the value):
      GroupNorm-apply (x - mean) rstd gamma + beta with the same fp32 stats on both sides: 4 roundings per side,
        E_gn = 2 gam(4) (|x - mean| rstd |gamma| + |beta|);
      SiLU f / (1 + e^-f): slope <= 1.1; the kernel's __expf is within 2 + 1.16|f| ulp and __fdividef within 2 ulp
        (CUDA programming guide), torch's sigmoid within 4 ulp: + |silu(f)| (10 + 1.16 |f|) 2^-23.
    Without either the value is copied: E = 0 (exact)."""
    xd = _d(x)
    C = xd.shape[-1]
    if stats is None and not silu:
        e = torch.zeros_like(xd)
    else:
        f, e = xd, torch.zeros_like(xd)
        if stats is not None:
            cg = C // groups
            st = _d(stats)
            mean = st[..., 0].repeat_interleave(cg, dim=1)[:, None, None, None, :]
            rstd = st[..., 1].repeat_interleave(cg, dim=1)[:, None, None, None, :]
            f = (xd - mean) * rstd * _d(gamma) + _d(beta)
            e = 2 * gam(4) * ((xd - mean).abs() * rstd * _d(gamma).abs() + _d(beta).abs())
        if silu:
            e = 1.1 * e + (f * torch.sigmoid(f)).abs() * (10 + 1.16 * f.abs()) * 2.0 ** -23
    # the double's own layout arithmetic carries E to the output positions (padding channels get 0); E is stored in bf16
    # on the way, rounded by < 2^-8 relative, which the factor 1 + 2^-7 undoes
    return _quiet(lambda: F_.vae_prep(e.float().to(torch.bfloat16), up=up, pad=pad, cp=cp)).double() * (1 + 2.0 ** -7)


def err_cfg_euler(cond, uncond, uncond2, x, *, g_txt, g_img=1.0, g_img_map=None, dt, **_):
    """x + dt (u2 + gi (u - u2) + gt (c - u)): 8 fp32 operations, plus the fp32 conversion of the three scalars:
    E = 2 gam(12) (|x| + |dt| (|u2| + |gi| (|u| + |u2|) + |gt| (|c| + |u|)))."""
    c, u, xx = _d(cond).abs(), _d(uncond).abs(), _d(x).abs()
    if uncond2 is None:
        m = u + abs(g_txt) * (c + u)
    else:
        u2 = _d(uncond2).abs()
        gi = abs(g_img) if g_img_map is None else _d(g_img_map).abs().reshape(-1).repeat(xx.numel() // g_img_map.numel()).view_as(xx)
        m = u2 + gi * (u + u2) + abs(g_txt) * (c + u)
    return 2 * gam(12) * (xx + abs(dt) * m)


def err_rf_masked_step(vc, vu, z, frame_mask, t_cur, t_next, *, guidance, noise=None, update=True, num_timesteps=1000, **_):
    """Per frame, as include/osb200.h osb_rf_masked_step: updated frames z + dt (u + g (c - u)) (E = 2 gam(8) M), re-noised
    frames (1 - a) z + a n (E = 2 gam(4) M), frames left alone E = 0 (bit-identical)."""
    N = float(num_timesteps)
    m = frame_mask.cpu() * N
    zz = _d(z).abs()
    e = torch.zeros_like(zz)
    tc, tn = t_cur.cpu(), t_next.cpu()
    fr = lambda f: f[:, None, :, None, None].expand_as(zz)  # noqa: E731
    if update:
        upd = m >= tc[:, None]
        dt = ((tc - tn) * (1.0 / N)).double()[:, None, None, None, None]
        mu = zz + dt.abs() * (_d(vu).abs() + abs(guidance) * (_d(vc).abs() + _d(vu).abs()))
        e = torch.where(fr(upd), 2 * gam(8) * mu, e)
        prev = upd
    else:
        prev = frame_mask.cpu() == 1
    if noise is not None:
        add = (m >= tn[:, None]) & ~prev
        a = (tn * (1.0 / N)).double()[:, None, None, None, None]
        e = torch.where(fr(add), 2 * gam(4) * ((1 - a).abs() * zz + a.abs() * _d(noise).abs()), e)
    return e


def err_head_tiles(a, w, bias, tmap, H, D, *, nkinds, norm_w=(), rope=None, rope_kinds=0, eps=1e-6):
    """[N // (H D), M, H D] budgets of the head-tile contents.  The accumulator is a GEMM (E_v = gam2(K + 1) Mv, see
    err_gemm); then per head row, in fp32 on both sides,
      RMSNorm x r w, r = (sum x^2 / D + eps)^-1/2: d(sum x^2) <= sum 2 |x| E_v + 2 gam(D) sum x^2, relative error of r
        eps_r <= d(sum x^2) / (2 (sum x^2 + D eps)) + 6u, E_n = r |w| E_v + |x r w| eps_r + 2 gam(3) |x r w|;
      RoPE (a c - b s, b c + a s) with the same fp32 tables: E_a' = |c| E_a + |s| E_b + 2 gam(2) (|a c| + |b s|)."""
    ad, wd = _d(a), _d(w)
    M, K = ad.shape
    v = ad @ wd.t()
    mv = ad.abs() @ wd.abs().t()
    if bias is not None:
        v, mv = v + _d(bias), mv + _d(bias).abs()
    ev = gam2(K + 1) * mv
    Cc = H * D
    _, pos = F_._seq_pos(tmap, M, "cpu")
    outs = []
    for kidx in range(wd.shape[0] // Cc):
        kind = kidx % nkinds
        x = v[:, kidx * Cc:(kidx + 1) * Cc].reshape(M, H, D)
        e = ev[:, kidx * Cc:(kidx + 1) * Cc].reshape(M, H, D)
        nw = norm_w[kind] if kind < len(norm_w) else None
        if nw is not None:
            ss = x.pow(2).sum(-1, keepdim=True)
            dss = (2 * x.abs() * e).sum(-1, keepdim=True) + 2 * gam(D) * ss
            eps_r = dss / (2 * (ss + D * eps)) + 6 * U
            r = (ss / D + eps).rsqrt()
            y = x * r * _d(nw)
            e = r * _d(nw).abs() * e + y.abs() * (eps_r + 2 * gam(3))
            x = y
        if rope is not None and (rope_kinds >> kind) & 1:
            c, s = _d(rope[0])[pos][:, None, :], _d(rope[1])[pos][:, None, :]
            xa, xb, ea, eb = x[..., 0::2], x[..., 1::2], e[..., 0::2], e[..., 1::2]
            na = c.abs() * ea + s.abs() * eb + 2 * gam(2) * ((xa * c).abs() + (xb * s).abs())
            nb_ = c.abs() * eb + s.abs() * ea + 2 * gam(2) * ((xb * c).abs() + (xa * s).abs())
            e = torch.stack((na, nb_), dim=-1).reshape(M, H, D)
        outs.append(e.reshape(M, Cc))
    return outs


def err_attn_tiles(qd, kd, vd, tmap_q, tmap_k, H, D, Lk, num_seqs, kv_lens=None, softmax_scale=None, out_map=None,
                   out_shape=None):
    """E for osb_attn_tiles from the dense operands the kernel read (see _attn_eps); (P |V|) and S are computed here in
    fp64 from the same operands."""
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    q, k, v = _d(qd), _d(kd), _d(vd)
    seq_q, pos_q = F_._seq_pos(tmap_q, q.shape[0], "cpu")
    seq_k, pos_k = F_._seq_pos(tmap_k, k.shape[0], "cpu")
    out_rows = torch.arange(q.shape[0])
    if out_map is not None:
        so, po = F_._seq_pos(out_map, q.shape[0], "cpu")
        inv = torch.empty(q.shape[0], dtype=torch.long)
        inv[so * tmap_q.L + po] = torch.arange(q.shape[0])
        out_rows = inv[seq_q * tmap_q.L + pos_q]
    e = torch.zeros(out_shape, dtype=torch.float64)
    qn = q.view(-1, H, D).norm(dim=-1).max()
    kn = k.view(-1, H, D).norm(dim=-1).max()
    eps = _attn_eps(D, (tmap_q.G if tmap_q.G > 1 else 1) * Lk, float(scale * qn * kn))
    for s in range(num_seqs):
        rq = (seq_q == s).nonzero().flatten()
        rk = (seq_k == s).nonzero().flatten()
        rk = rk[pos_k[rk].argsort()]
        n = Lk if kv_lens is None else min(int(kv_lens[s]), Lk)
        if n <= 0:
            continue
        rk = rk[:n]
        qq = q[rq].view(-1, H, D).transpose(0, 1)
        kk = k[rk].view(-1, H, D).transpose(0, 1)
        vv = v[rk].view(-1, H, D).transpose(0, 1).abs()
        p = torch.softmax(qq @ kk.transpose(-1, -2) * scale, dim=-1)
        e[out_rows[rq], : H * D] = (eps * (p @ vv)).transpose(0, 1).reshape(len(rq), H * D)
    return e


# ===================================================================================================================
# hand-picked cases: the argument combinations where the two could disagree on a convention
# ===================================================================================================================
@pytest.mark.parametrize("C,G,mode", [(64, 1, "rows"), (1152, 3, "rows"), (200, 4, "mod_index"), (8192, 2, "rows"),
                                      (384, 2, "scatter3")])
def test_ln_modulate(C, G, mode):
    import osb200 as osb

    dev = _dev()
    g = _gen(C + G)
    rows = 96
    x = _bf(rows, C, g=g)
    x[5] += 40.0                                    # one row with a large mean
    x = x.to(torch.bfloat16)
    table = torch.randn(G, 2 * C + 8, generator=g) * 0.3    # shift | scale as views of one wider table (row stride)
    shift, scale = table[:, :C], table[:, C + 8:2 * C + 8]
    kw = dict(group_rows=rows // G if mode != "mod_index" else rows // 8, eps=1e-5 if C == 200 else 1e-6)
    if mode == "mod_index":
        kw["mod_index"] = torch.randint(0, G, (8,), generator=g, dtype=torch.int32)
    xc, sc, hc = x.to(dev), scale.to(dev), shift.to(dev)
    kwd = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    if mode == "scatter3":
        I, J = 8, rows // 8
        buf_k = torch.full((rows, C), float("nan"), dtype=torch.bfloat16, device=dev)
        buf_d = torch.full((rows, C), float("nan"), dtype=torch.bfloat16)
        _launches(osb, lambda: osb.ln_modulate(xc, hc, sc, scatter=osb.make_scatter(3, 1, 0, I, J, [buf_k]), **kwd),
                  lambda: F_.ln_modulate(x, shift, scale, scatter=F_.make_scatter(3, 1, 0, I, J, [buf_d]), **kw))
        plain = osb.ln_modulate(xc, hc, sc, **kwd)
        routed = plain.view(1, I, J, C).transpose(1, 2).reshape(rows, C)
        _check(f"ln_modulate scatter mode 3 routing C={C}", buf_k, routed)
        e = err_ln(x, shift, scale, **kw).view(1, I, J, C).transpose(1, 2).reshape(rows, C)
        _check(f"ln_modulate scatter mode 3 C={C}", buf_k, buf_d, e)
        return
    out_k, out_d = _launches(osb, lambda: osb.ln_modulate(xc, hc, sc, **kwd), lambda: F_.ln_modulate(x, shift, scale, **kw))
    _check(f"ln_modulate C={C} G={G} {mode}", out_k, out_d, err_ln(x, shift, scale, **kw))


GEMM_CASES = [
    # M, N, K, epilogue, gate mode, residual mode, A slice, block_n
    (300, 72, 200, 0, None, None, False, 0),
    (300, 72, 200, 1, None, None, True, 64),
    (300, 200, 200, 2, "rows", "alias", False, 128),
    (257, 392, 136, 2, "mod_index", "sep", True, 192),
    (130, 520, 64, 2, None, "alias", False, 256),
    (64, 264, 200, 1, None, None, False, 256),
    (200, 256, 520, 2, "rows", None, True, 0),
]


def _gemm_inputs(M, N, K, epi, gate_mode, res_mode, a_slice, seed):
    g = _gen(seed)
    wide = _bf(M, K + 24, g=g)
    a = wide[:, 16:16 + K] if a_slice else wide[:, :K].contiguous()
    w = _bf(N, K, g=g, scale=K ** -0.5)
    bias = _bf(N, g=g, scale=0.1)
    kw = dict(epilogue=epi)
    if epi == 2:
        if gate_mode == "rows":
            kw.update(gate=(torch.randn(3, N + 4, generator=g))[:, :N], group_rows=-(-M // 3))
        elif gate_mode == "mod_index":
            kw.update(gate=torch.randn(4, N, generator=g), group_rows=-(-M // 5),
                      mod_index=torch.tensor([3, 0, 2, 1, 3], dtype=torch.int32))
        if res_mode is not None:
            kw["residual"] = _bf(M, N, g=g)
    return a, w, bias, kw


def _to(kw, dev):
    return {k: (_slice_to(v, dev) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}


def _with_slack(x, dev, slack_elems=64):
    """x on the device followed by zeroed slack, as osb200.vae_prep allocates it: narrow-mode convolution windows read
    up to 64 - Cp elements past the last position."""
    buf = torch.zeros(x.numel() + slack_elems, dtype=x.dtype, device=dev)
    buf[: x.numel()].copy_(x.reshape(-1))
    return buf[: x.numel()].view(x.shape)


def _slice_to(t, dev):
    """Move a (possibly column-sliced) CPU tensor to the device keeping its strides (the kernel sees the same view)."""
    if t._base is None:
        return t.to(dev)
    base = t._base.to(dev)
    return base.as_strided(t.shape, t.stride(), t.storage_offset())


@pytest.mark.parametrize("case", GEMM_CASES, ids=[f"M{c[0]}N{c[1]}K{c[2]}e{c[3]}{c[4]}{c[5]}bn{c[7]}" for c in GEMM_CASES])
@pytest.mark.parametrize("rank", [0, 8, 72])
def test_gemm_and_lora(case, rank):
    import osb200 as osb

    dev = _dev()
    M, N, K, epi, gate_mode, res_mode, a_slice, bn = case
    a, w, bias, kw = _gemm_inputs(M, N, K, epi, gate_mode, res_mode, a_slice, seed=M + N + K + rank)
    err = None
    if rank:
        g = _gen(rank)
        u = _bf(M, rank + 8, g=g)[:, 8:]                      # U as a column slice (row stride free)
        b = _bf(N, rank, g=g, scale=0.3 / rank ** 0.5)
        err = err_gemm(a, w, bias, u=u, b=b, **kw)
    else:
        err = err_gemm(a, w, bias, **kw)
    kd, kc = dict(kw), _to(kw, dev)
    if res_mode == "alias":                                  # out is the residual stream itself
        kd["out"] = kd["residual"] = kw["residual"].clone()
        kc["out"] = kc["residual"]
    ac, wc, bc = _slice_to(a, dev), w.to(dev), bias.to(dev)
    if rank:
        uc, bcl = _slice_to(u, dev), b.to(dev)
        out_k, out_d = _launches(osb, lambda: osb.gemm_lora(ac, wc, bc, uc, bcl, block_n=bn, **kc),
                                 lambda: F_.gemm_lora(a, w, bias, u, b, block_n=bn, **kd))
    else:
        out_k, out_d = _launches(osb, lambda: osb.gemm(ac, wc, bc, block_n=bn, **kc), lambda: F_.gemm(a, w, bias, block_n=bn, **kd))
    if res_mode == "alias":
        assert out_k.data_ptr() == kc["residual"].data_ptr() and out_d.data_ptr() == kd["residual"].data_ptr()
    _check(f"{'gemm_lora r=%d' % rank if rank else 'gemm'} {M}x{N}x{K} epi={epi} gate={gate_mode} res={res_mode} "
           f"slice={a_slice} bn={bn}", out_k, out_d, err)


def _rope_tables(L, D, theta=10000.0):
    inv = 1.0 / (theta ** (torch.arange(0, D, 2).float() / D))
    ang = torch.arange(L).float()[:, None] * inv[None] * 0.37
    return ang.cos().contiguous(), ang.sin().contiguous()


def _attn_short_case(name, seed):
    """(tensors, kwargs) of one osb_attn_short call laid out as the host code lays it out."""
    g = _gen(seed)
    if name == "spatial":              # STDiT3 spatial: sequences = frames, tokens contiguous; q/k/v column slices of qkv
        B, T, S, H, D = 1, 2, 200, 2, 72
        C = H * D
        qkv = _bf(B * T * S, 3 * C, g=g)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        kw = dict(num_seqs=B * T, seqs_per_batch=T, q_strides=(T * S, S, 1), k_strides=(T * S, S, 1), Lq=S, Lk=S,
                  num_heads=H, head_dim=D, q_norm_w=_bf(D, g=g, scale=0.2) + 1, k_norm_w=_bf(D, g=g, scale=0.2) + 1)
        out = torch.zeros(B * T * S, C, dtype=torch.bfloat16)
    elif name == "temporal":           # STDiT3 temporal: sequences along T (token stride S), packed (Lq = 24 -> G = 5)
        B, T, S, H, D = 2, 24, 5, 2, 64
        C = H * D
        qkv = _bf(B * T * S, 3 * C, g=g)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        cos, sin = _rope_tables(T, D)
        kw = dict(num_seqs=B * S, seqs_per_batch=S, q_strides=(T * S, 1, S), k_strides=(T * S, 1, S), Lq=T, Lk=T,
                  num_heads=H, head_dim=D, rope_cos=cos, rope_sin=sin)
        out = torch.zeros(B * T * S, C, dtype=torch.bfloat16)
    elif name == "cross":              # cross-attention: Lk != Lq, kv_lens including 0, k | v one kv buffer
        B, N, Ly, H, D = 3, 150, 40, 2, 72
        C = H * D
        q = _bf(B * N, C, g=g)
        kv = _bf(B * Ly, 2 * C, g=g)
        k, v = kv[:, :C], kv[:, C:]
        kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(N, 0, 1), k_strides=(Ly, 0, 1), Lq=N, Lk=Ly, num_heads=H,
                  head_dim=D, kv_lens=torch.tensor([40, 13, 0], dtype=torch.int32), softmax_scale=0.09)
        out = torch.zeros(B * N, C, dtype=torch.bfloat16)
    elif name == "joint":              # MMDiT joint txt | img: two norm weight pairs split at the text length, rotate-half
        B, Lt, Li, H, D = 2, 32, 160, 2, 128
        L, C = Lt + Li, H * D
        qkv = _bf(B * L, 3 * C, g=g)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        cos, sin = _rope_tables(L, D)
        one = lambda: _bf(D, g=g, scale=0.2) + 1  # noqa: E731
        kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
                  head_dim=D, q_norm_w=one(), k_norm_w=one(), q_norm_w2=one(), k_norm_w2=one(), norm_split=Lt,
                  rope_cos=cos, rope_sin=sin, rope_half=True, softmax_scale=0.1, norm_eps=1e-5)
        out = torch.zeros(B * L, C, dtype=torch.bfloat16)
    elif name == "packed_kv_lens":     # packed short sequences (G = 6) with per-sequence key counts, rotate-half D = 64
        n, L, H, D = 9, 20, 2, 64
        C = H * D
        qkv = _bf(n * L, 3 * C, g=g)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        cos, sin = _rope_tables(L, D)
        kw = dict(num_seqs=n, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
                  head_dim=D, kv_lens=torch.tensor([20, 0, 7, 1, 20, 19, 3, 11, 16], dtype=torch.int32),
                  q_norm_w=_bf(D, g=g, scale=0.2) + 1, k_norm_w=_bf(D, g=g, scale=0.2) + 1, rope_cos=cos, rope_sin=sin,
                  rope_half=True)
        out = torch.zeros(n * L, C, dtype=torch.bfloat16)
    else:                              # interleaved RoPE at head_dim 128, Lq > 128 with a ragged last q tile
        B, L, H, D = 1, 300, 2, 128
        C = H * D
        qkv = _bf(B * L, 3 * C, g=g)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        cos, sin = _rope_tables(L, D)
        kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
                  head_dim=D, q_norm_w=_bf(D, g=g, scale=0.2) + 1, k_norm_w=_bf(D, g=g, scale=0.2) + 1, rope_cos=cos,
                  rope_sin=sin)
        out = torch.zeros(B * L, C, dtype=torch.bfloat16)
    return (q, k, v, out), kw


@pytest.mark.parametrize("name", ["spatial", "temporal", "cross", "joint", "packed_kv_lens", "rope128"])
def test_attn_short(name):
    import osb200 as osb

    dev = _dev()
    (q, k, v, out), kw = _attn_short_case(name, seed=len(name))
    err = err_attn_short(q, k, v, out, **kw)
    qc, kc_, vc = _slice_to(q, dev), _slice_to(k, dev), _slice_to(v, dev)
    out_k = out.to(dev)
    out_d = out.clone()
    kwc = _to(kw, dev)
    _launches(osb, lambda: osb.attn_short(qc, kc_, vc, out_k, **kwc), lambda: F_.attn_short(q, k, v, out_d, **kw))
    _check(f"attn_short {name}", out_k, out_d, err)


HT_CASES = [
    # name, map args (mode, L, S, T, kw), rows, H, D, nkinds, kind0, total kinds, kidx count, norm kinds, rope mask
    ("spatial-qkv", (0, 200, 0, 0, {}), 400, 2, 72, 3, 0, 3, 3, (0, 1), 0),
    ("temporal-packed-rope", (1, 24, 5, 24, {}), 240, 2, 64, 3, 0, 3, 3, (0, 1), 0b011),
    ("cross-q-kind0", (0, 150, 0, 0, {"pack": False}), 300, 2, 72, 1, 0, 1, 1, (), 0),
    ("keys-only-kv-blocks", (0, 40, 0, 0, {"keys_only": True}), 120, 2, 72, 2, 2, 6, 4, (0,), 0),
    ("four-kinds", (0, 128, 0, 0, {}), 256, 2, 128, 4, 1, 5, 4, (1, 3), 0b1010),
    ("mode1-unpacked-rope", (1, 100, 3, 100, {}), 300, 2, 64, 2, 0, 2, 2, (1,), 0b011),
]


def _head_tiles_case(case, seed, osb, dev):
    name, (mode, L, S, T, mkw), rows, H, D, nk, kind0, kinds, nkid, norm_kinds, rmask = case
    g = _gen(seed)
    tm = osb.tile_map(mode, L, S, T, **mkw)
    C = H * D
    K = 200
    a = _bf(rows, K, g=g)
    w = _bf(nkid * C, K, g=g, scale=K ** -0.5)
    bias = _bf(nkid * C, g=g, scale=0.1)
    norm_w = tuple((_bf(D, g=g, scale=0.2) + 1) if i in norm_kinds else None for i in range(nk))
    rope = _rope_tables(L, D) if rmask else None
    real = osb.HeadTiles(rows, tm, kinds, H, D, dev)
    fake = F_.HeadTiles(rows, tm, kinds, H, D, "cpu")
    kw = dict(nkinds=nk, norm_w=norm_w, rope=rope, rope_kinds=rmask, kind0=kind0)
    kwc = dict(kw, norm_w=tuple(None if t is None else t.to(dev) for t in norm_w),
               rope=None if rope is None else (rope[0].to(dev), rope[1].to(dev)))
    _launches(osb, lambda: osb.gemm_head_tiles(a.to(dev), w.to(dev), bias.to(dev), real, **kwc),
              lambda: F_.gemm_head_tiles(a, w, bias, fake, **kw))
    errs = err_head_tiles(a, w, bias, tm, H, D, nkinds=nk, norm_w=norm_w, rope=rope, rope_kinds=rmask)
    for kind in range(kinds):
        got = read_tiles(real, kind)
        if kind0 <= kind < kind0 + nkid:
            _check(f"head tiles {name} kind {kind}", got, fake.dense[kind], errs[kind - kind0])
        else:
            _check(f"head tiles {name} kind {kind} (not written: zero)", got, fake.dense[kind])
    return real, fake, tm


@pytest.mark.parametrize("case", HT_CASES, ids=[c[0] for c in HT_CASES])
def test_gemm_head_tiles(case):
    import osb200 as osb

    _head_tiles_case(case, 3, osb, _dev())


def _attn_tiles_run(osb, name, qt, kvt, q_kind, k_kind, v_kind, Lk, num_seqs, rows, C, min_identical=0.0, **kw):
    """The double attends over the DECODED kernel tiles, so the comparison isolates the attention itself.
    min_identical: lower limit on the bit-identical fraction (see the single-key-block cross case)."""
    dev = qt.buf.device
    H, D = qt.heads, qt.head_dim
    fq = F_.HeadTiles(qt.rows, qt.map, qt.kinds, H, D, "cpu")
    fkv = fq if kvt is qt else F_.HeadTiles(kvt.rows, kvt.map, kvt.kinds, H, D, "cpu")
    for t, f in ((qt, fq), (kvt, fkv)):
        for kind in range(t.kinds):
            f.dense[kind] = read_tiles(t, kind).cpu()
    out_k = torch.full((rows, C), float("nan"), dtype=torch.bfloat16, device=dev)
    out_d = torch.full((rows, C), float("nan"), dtype=torch.bfloat16)
    kwc = _to(kw, dev)
    _launches(osb, lambda: osb.attn_tiles(qt, kvt, out_k, q_kind=q_kind, k_kind=k_kind, v_kind=v_kind, Lk=Lk,
                                          num_seqs=num_seqs, **kwc),
              lambda: F_.attn_tiles(fq, fkv, out_d, q_kind=q_kind, k_kind=k_kind, v_kind=v_kind, Lk=Lk, num_seqs=num_seqs,
                                    **kw))
    err = err_attn_tiles(fq.dense[q_kind], fkv.dense[k_kind], fkv.dense[v_kind], fq.map, fkv.map, H, D, Lk, num_seqs,
                         kv_lens=kw.get("kv_lens"), softmax_scale=kw.get("softmax_scale"), out_map=kw.get("out_map"),
                         out_shape=(rows, C))
    _, same, n = _check(f"attn_tiles {name}", out_k, out_d, err)
    assert same / n >= min_identical, f"attn_tiles {name}: only {same / n:.4f} of the outputs are bit-identical"


def test_attn_tiles_self_packed_transposed_and_cross():
    import osb200 as osb

    dev = _dev()
    # spatial self-attention, ragged last tile, non-default scale
    qt, _, tm = _head_tiles_case(HT_CASES[0], 5, osb, dev)
    _attn_tiles_run(osb, "spatial L=200", qt, qt, 0, 1, 2, 200, 2, 400, 144, softmax_scale=0.1)
    # temporal, packed (G = 5) with RoPE
    qt, _, tm = _head_tiles_case(HT_CASES[1], 6, osb, dev)
    _attn_tiles_run(osb, "temporal packed T=24", qt, qt, 0, 1, 2, 24, 10, 240, 128)
    # tiles written from a transposed [B, S, T] stream (mode 0), output rows frame-major (out_map mode 1)
    B, T, S, H, D = 2, 24, 5, 2, 64
    case = ("transposed", (0, T, 0, 0, {}), B * S * T, H, D, 3, 0, 3, 3, (0, 1), 0)
    qt, _, _ = _head_tiles_case(case, 7, osb, dev)
    _attn_tiles_run(osb, "temporal out_map", qt, qt, 0, 1, 2, T, B * S, B * S * T, H * D, out_map=osb.tile_map(1, T, S, T))
    # cross-attention: unpacked queries, keys-only text tiles of several blocks, kv_lens with 0
    qcase = ("cross-q", (0, 150, 0, 0, {"pack": False}), 450, 2, 72, 1, 0, 1, 1, (), 0)
    kcase = ("cross-kv", (0, 40, 0, 0, {"keys_only": True}), 120, 2, 72, 2, 0, 4, 4, (), 0)
    qt, _, _ = _head_tiles_case(qcase, 8, osb, dev)
    kt, _, _ = _head_tiles_case(kcase, 9, osb, dev)
    lens = torch.tensor([40, 0, 17], dtype=torch.int32)
    _attn_tiles_run(osb, "cross kv_lens block 1", qt, kt, 0, 2, 3, 40, 3, 450, 144, kv_lens=lens)
    # Lk = 40 keys fit one 64-key block, so the kernel's running max is the final max and both sides round the same fp32
    # P: measured 0.9997 of the outputs bit-identical on the H100.  Rounding the NORMALISED P instead (the convention
    # the double once used) agrees on only ~0.52 of them, which the Higham-style bound above cannot see (both conventions
    # are within 2^-8 of the exact P).  0.9 separates the two.
    _attn_tiles_run(osb, "cross no kv_lens D=72", qt, kt, 0, 0, 1, 40, 3, 450, 144, min_identical=0.9, softmax_scale=0.2)
    # head_dim 128, four kinds, attention over kinds 1 | 3 | 4
    qt, _, _ = _head_tiles_case(HT_CASES[4], 10, osb, dev)
    _attn_tiles_run(osb, "D=128 kinds 1,3,4", qt, qt, 1, 3, 4, 128, 2, 256, 256)


def err_group_stats(x, groups, eps=1e-6):
    """fp32 outputs (no bf16 rounding): both sum fp32 values over n = positions * C / groups elements.
      mean: the kernel sums x - K (K the group's first element), the double x:
            |d mean| <= gam(n) (mean|x - K| + mean|x|) + 2u |mean| (the final roundings), plus the fp32 ulp of _check;
      var:  kernel E[d^2] - E[d]^2 from fp32 sums, |d var_k| <= gam(n) (E[d^2] + 2 |E d| E|d|); the double's two-pass
            mean((x - m')^2) is var + (m' - m)^2 within gam(n + 2) (var + dm^2), dm = gam(n) mean|x|;
      rstd: relative error (d var_k + d var_d) / (2 (var + eps)) + 4u."""
    nb, C = x.shape[0], x.shape[-1]
    xd = _d(x).reshape(nb, -1, groups, C // groups)
    n = xd.shape[1] * xd.shape[3]
    d = xd - xd[:, :1, :, :1]
    mean = xd.mean(dim=(1, 3))
    var = (xd - mean[:, None, :, None]).pow(2).mean(dim=(1, 3))
    e_mean = gam(n) * (d.abs().mean(dim=(1, 3)) + xd.abs().mean(dim=(1, 3))) + 2 * U * mean.abs()
    dm = gam(n) * xd.abs().mean(dim=(1, 3))
    dvk = gam(n) * (d.pow(2).mean(dim=(1, 3)) + 2 * d.mean(dim=(1, 3)).abs() * d.abs().mean(dim=(1, 3)))
    dvd = gam(n + 2) * (var + dm ** 2) + dm ** 2
    rstd = (var + eps).rsqrt()
    return torch.stack((e_mean, rstd * ((dvk + dvd) / (2 * (var + eps)) + 4 * U)), dim=-1)


def test_group_stats():
    """Two batch entries, 3 x 40 x 30 = 3600 positions (two 2048-position chunks), one group with mean 50 >> std
    (a one-pass fp32 E[x^2] - E[x]^2 would lose its variance)."""
    import osb200 as osb

    dev = _dev()
    g = _gen(17)
    nb, T, H, W, C, G = 2, 3, 40, 30, 64, 8
    x = torch.randn(nb, T, H, W, C, generator=g)
    x[..., 24:32] += 50.0
    x = x.to(torch.bfloat16)
    got, want = _launches(osb, lambda: osb.group_stats(x.to(dev), G, eps=1e-6), lambda: F_.group_stats(x, G, eps=1e-6))
    e = err_group_stats(x, G, 1e-6)
    _check("group_stats mean", got[..., 0], want[..., 0], e[..., 0], ulp=ulp_fp32)
    _check("group_stats rstd", got[..., 1], want[..., 1], e[..., 1], ulp=ulp_fp32)


VAE_UP = list(itertools.product((1, 2), repeat=3))
VAE_PAD = [(0, 0, 0), (2, 1, 1), (1, 0, 1), (0, 1, 0)]


@pytest.mark.parametrize("norm", ["copy", "silu", "gn", "gn+silu"])
def test_vae_prep(norm):
    """Every up-sampling x padding combination, cp > c.  Copy / up-sampling / replicate padding, the zero channels c..cp
    and the zeroed slack after the buffer are exact; GroupNorm / SiLU are one rounding (err_vae_prep)."""
    import osb200 as osb

    dev = _dev()
    g = _gen(23)
    nb, T, H, W, C, G, cp = 2, 3, 5, 6, 16, 4, 24
    x = _bf(nb, T, H, W, C, g=g)
    stats = gamma = beta = None
    if "gn" in norm:
        stats = F_.group_stats(x, G)
        gamma, beta = _bf(C, g=g, scale=0.3) + 1, _bf(C, g=g, scale=0.2)
    silu = "silu" in norm
    for up in VAE_UP:
        for pad in VAE_PAD:
            kw = dict(stats=stats, gamma=gamma, beta=beta, groups=G, silu=silu, up=up, pad=pad, cp=cp)
            got, want = _launches(osb, lambda: osb.vae_prep(x.to(dev), **_to(kw, dev)), lambda: F_.vae_prep(x, **kw))
            tag = f"vae_prep {norm} up={up} pad={pad}"
            e = err_vae_prep(x, **kw)
            _check(tag, got[..., :C], want[..., :C], None if norm == "copy" else e[..., :C])
            _check(tag + " channels c..cp", got[..., C:], want[..., C:])
            slack = got._base[got.numel():]
            _check(tag + " slack", slack, torch.zeros_like(slack))


CONV_CASES = [
    # narrow, Cin, Cp, Cout, taps, stride, residual, block_n
    (False, 40, 64, 72, (3, 3, 3), (1, 1, 1), True, 0),
    (False, 64, 64, 64, (3, 3, 3), (1, 2, 2), False, 64),
    (False, 128, 128, 200, (3, 3, 3), (2, 2, 2), False, 128),
    (False, 64, 64, 192, (1, 3, 3), (1, 1, 1), True, 192),
    (False, 64, 64, 264, (1, 3, 3), (1, 2, 2), False, 256),
    (True, 3, 8, 64, (3, 3, 3), (1, 1, 1), False, 0),
    (True, 12, 16, 72, (3, 3, 3), (1, 2, 2), True, 128),
    (True, 3, 16, 32, (1, 3, 3), (2, 2, 2), False, 64),
]


@pytest.mark.parametrize("case", CONV_CASES, ids=[f"{'narrow' if c[0] else 'normal'}-cp{c[2]}-co{c[3]}-k{c[4][0]}-s{''.join(map(str, c[5]))}"
                                                  f"-{'res' if c[6] else 'nores'}-bn{c[7]}" for c in CONV_CASES])
def test_pack_conv_weight_and_conv3d(case):
    import osb200 as osb

    dev = _dev()
    narrow, cin, cp, cout, taps, stride, res, bn = case
    g = _gen(cin + cout)
    kt, kh, kw_ = taps
    w = torch.randn(cout, cin, kt, kh, kw_, generator=g) * (cin * kt * kh * kw_) ** -0.5
    wp_k = osb.pack_conv_weight(w.to(dev), cp, narrow)
    wp_d = F_.pack_conv_weight(w, cp, narrow)
    _check(f"pack_conv_weight narrow={narrow} cp={cp} taps={taps}", wp_k, wp_d)
    nb, T, H, W = 2, 5, 9, 10
    x = torch.zeros(nb, T, H, W, cp, dtype=torch.bfloat16)      # channels zero-padded to Cp, as the VAE stores them
    x[..., :cin] = _bf(nb, T, H, W, cin, g=g)
    pad = (kt - 1, kh // 2, kw_ // 2)
    x_pad = F_.vae_prep(x, pad=pad)
    tp, hp, wp = x_pad.shape[1:4]
    out_thw = tuple((n - k) // s + 1 for n, k, s in zip((tp, hp, wp), taps, stride))
    bias = _bf(cout, g=g, scale=0.1)
    residual = _bf(nb, *out_thw, cout, g=g) if res else None
    kw = dict(out_thw=out_thw, stride=stride, taps=taps, narrow=narrow, residual=residual, block_n=bn)
    xk = _with_slack(x_pad, dev)
    got, want = _launches(osb, lambda: osb.conv3d(xk, wp_k, bias.to(dev), **_to(kw, dev)),
                          lambda: F_.conv3d(x_pad, wp_d, bias, **kw))
    _check(f"conv3d narrow={narrow} cp={cp} cout={cout} taps={taps} stride={stride} res={res} bn={bn}", got, want,
           err_conv(x_pad, wp_d, bias, **kw))


@pytest.mark.parametrize("mode", ["two", "three", "map"])
def test_cfg_euler(mode):
    import osb200 as osb

    dev = _dev()
    g = _gen(31)
    shape = (2, 16, 3, 6, 8)
    c, u, u2, x = (_bf(*shape, g=g) for _ in range(4))
    kw = dict(g_txt=6.5, dt=-0.0345)
    if mode == "two":
        u2 = None
    elif mode == "three":
        kw["g_img"] = 2.25
    else:
        kw["g_img_map"] = _bf(6 * 8 * 4, g=g)       # period 192 elements, repeats over the latent
    got, want = _launches(osb, lambda: osb.cfg_euler(c.to(dev), u.to(dev), None if u2 is None else u2.to(dev), x.to(dev),
                                                     **_to(kw, dev)),
                          lambda: F_.cfg_euler(c, u, u2, x, **kw))
    _check(f"cfg_euler {mode}", got, want, err_cfg_euler(c, u, u2, x, **kw))


@pytest.mark.parametrize("update,noise,HW,in_place", [(True, False, (4, 6), False), (True, True, (4, 6), True),
                                                      (False, True, (4, 6), False), (True, True, (3, 5), False),
                                                      (False, True, (3, 5), True)])
def test_rf_masked_step(update, noise, HW, in_place):
    import osb200 as osb

    dev = _dev()
    g = _gen(37)
    B, C, T = 2, 4, 6
    shape = (B, C, T) + HW
    vc, vu, z, nz = (_bf(*shape, g=g) for _ in range(4))
    fm = torch.tensor([[0.0, 0.5, 1.0, 1.0, 0.3, 1.0], [1.0, 1.0, 0.0, 0.7, 1.0, 0.45]])
    tc, tn = torch.tensor([600.0, 800.0]), torch.tensor([400.0, 650.0])
    kw = dict(guidance=4.5, noise=nz if noise else None, update=update)
    err = err_rf_masked_step(vc, vu, z, fm, tc, tn, **kw)
    zk, zd = z.to(dev), z.clone()
    kwc = _to(kw, dev)
    args_k = (vc.to(dev), vu.to(dev), zk, fm.to(dev), tc.to(dev), tn.to(dev))
    got, want = _launches(osb, lambda: osb.rf_masked_step(*args_k, out=zk if in_place else None, **kwc),
                          lambda: F_.rf_masked_step(vc, vu, zd, fm, tc, tn, out=zd if in_place else None, **kw))
    if in_place:
        assert got.data_ptr() == zk.data_ptr() and want.data_ptr() == zd.data_ptr()
    tag = f"rf_masked_step update={update} noise={noise} HW={HW} in_place={in_place}"
    left = (err == 0).all(dim=(1, 3, 4))                                    # [B, T]: frames the step leaves alone
    sel = left[:, None, :, None, None].expand(shape)
    _check(tag + " frames left alone", got.cpu()[sel], want[sel])
    _check(tag, got, want, err)


# ===================================================================================================================
# refusals: every invalid call raises OsbError from both implementations (and launches nothing)
# ===================================================================================================================
def _refusals():
    b = lambda *s: torch.zeros(*s, dtype=torch.bfloat16)  # noqa: E731
    f = lambda *s: torch.zeros(*s, dtype=torch.float32)  # noqa: E731
    cos, sin = f(8, 36), f(8, 36)
    qkv = b(8, 3 * 144)
    attn = dict(num_seqs=1, seqs_per_batch=1, q_strides=(8, 0, 1), k_strides=(8, 0, 1), Lq=8, Lk=8, num_heads=2)
    x5 = b(1, 2, 4, 4, 16)
    return [
        ("rotate-half RoPE with head_dim 72", lambda m, d: m.attn_short(*(t.to(d) for t in (qkv[:, :144], qkv[:, 144:288], qkv[:, 288:], b(8, 144))),
                                                                         head_dim=72, rope_cos=cos.to(d), rope_sin=sin.to(d), rope_half=True, **attn)),
        ("conv3d taps 4", lambda m, d: m.conv3d(b(1, 6, 6, 6, 64).to(d), b(64, 4 * 9 * 64).to(d), None, out_thw=(1, 4, 4), taps=(4, 3, 3))),
        ("conv3d taps 0", lambda m, d: m.conv3d(b(1, 6, 6, 6, 64).to(d), b(64, 9 * 64).to(d), None, out_thw=(4, 4, 4), taps=(0, 3, 3))),
        ("conv3d stride 3", lambda m, d: m.conv3d(b(1, 9, 6, 6, 64).to(d), b(64, 27 * 64).to(d), None, out_thw=(3, 4, 4), stride=(3, 1, 1))),
        ("conv3d Cp 32", lambda m, d: m.conv3d(b(1, 6, 6, 6, 32).to(d), b(64, 27 * 32).to(d), None, out_thw=(4, 4, 4))),
        ("conv3d narrow Cp 32", lambda m, d: m.conv3d(b(1, 6, 6, 6, 32).to(d), b(64, 9 * 64).to(d), None, out_thw=(4, 4, 4), narrow=True)),
        ("vae_prep up 3", lambda m, d: m.vae_prep(x5.to(d), up=(1, 3, 1))),
        ("vae_prep up 4", lambda m, d: m.vae_prep(x5.to(d), up=(4, 1, 1))),
        ("ln_modulate C % 8", lambda m, d: m.ln_modulate(b(4, 12).to(d), f(1, 12).to(d), f(1, 12).to(d), group_rows=4)),
        ("ln_modulate C > 8192", lambda m, d: m.ln_modulate(b(2, 8200).to(d), f(1, 8200).to(d), f(1, 8200).to(d), group_rows=2)),
        ("gemm_head_tiles nkinds 5", lambda m, d: m.gemm_head_tiles(b(64, 64).to(d), b(5 * 128, 64).to(d), None,
                                                                    (osb_ht(m, d, 64, m.tile_map(0, 64), 5, 2, 64)), nkinds=5)),
        ("gemm K % 8", lambda m, d: m.gemm(b(16, 12).to(d), b(16, 12).to(d))),
        ("gemm N % 8", lambda m, d: m.gemm(b(16, 16).to(d), b(12, 16).to(d))),
        ("gemm_lora r % 8", lambda m, d: m.gemm_lora(b(16, 16).to(d), b(16, 16).to(d), None, b(16, 4).to(d), b(16, 4).to(d))),
        ("group_stats C/8 not dividing 256", lambda m, d: m.group_stats(b(1, 2, 4, 4, 24).to(d), 3)),
        ("cfg_euler n % 8", lambda m, d: m.cfg_euler(*(b(12).to(d) for _ in range(2)), None, b(12).to(d), g_txt=1.0, dt=0.1)),
        ("attn_tiles kv_lens with packed q map", lambda m, d: m.attn_tiles(osb_ht(m, d, 64, m.tile_map(0, 16), 3, 2, 64),
                                                                           osb_ht(m, d, 64, m.tile_map(0, 16), 3, 2, 64),
                                                                           b(64, 128).to(d), Lk=16, num_seqs=4,
                                                                           kv_lens=torch.full((4,), 16, dtype=torch.int32).to(d))),
    ] + _shape_refusals()


def _shape_refusals():
    """Wrong-shaped optional GEMM operands (out, bias, residual, gate, mod_index) and a K mismatch.  Each wrong-shaped
    tensor is a view into an allocation large enough for what a launch would touch, so a missing check shows as "did
    not raise", never as an out-of-bounds access."""
    b = lambda *s: torch.zeros(*s, dtype=torch.bfloat16)  # noqa: E731
    f = lambda *s: torch.zeros(*s, dtype=torch.float32)  # noqa: E731
    e = lambda *s: torch.zeros(*s, dtype=torch.float8_e4m3fn)  # noqa: E731
    gr = dict(epilogue=F_.EPI_BIAS_GATE_RES, group_rows=8)
    lo = lambda d: (b(16, 8).to(d), b(16, 8).to(d))  # noqa: E731   u [M, r], b [N, r]
    s8 = lambda d: (f(16).to(d) + 1, f(16).to(d) + 1)  # noqa: E731   a_scale [M], w_scale [N]
    return [
        ("gemm out [M, N-8]", lambda m, d: m.gemm(b(16, 16).to(d), b(16, 16).to(d), out=b(16, 16).to(d)[:, :8])),
        ("gemm bias [N-8]", lambda m, d: m.gemm(b(16, 16).to(d), b(16, 16).to(d), b(16).to(d)[:8])),
        ("gemm residual [M-1, N]", lambda m, d: m.gemm(b(16, 16).to(d), b(16, 16).to(d), residual=b(16, 16).to(d)[:15],
                                                       epilogue=F_.EPI_BIAS_GATE_RES)),
        ("gemm gate [G, N-8]", lambda m, d: m.gemm(b(16, 16).to(d), b(16, 16).to(d), gate=f(2, 16).to(d)[:, :8], **gr)),
        ("gemm gate rows < groups", lambda m, d: m.gemm(b(16, 16).to(d), b(16, 16).to(d), gate=f(2, 16).to(d)[:1], **gr)),
        ("gemm mod_index short", lambda m, d: m.gemm(b(16, 16).to(d), b(16, 16).to(d), gate=f(2, 16).to(d),
                                                     mod_index=torch.zeros(2, dtype=torch.int32).to(d)[:1], **gr)),
        ("gemm K mismatch", lambda m, d: m.gemm(b(16, 16).to(d), b(16, 24).to(d))),
        ("gemm_lora out [M-1, N]", lambda m, d: m.gemm_lora(b(16, 16).to(d), b(16, 16).to(d), None, *lo(d),
                                                            out=b(16, 16).to(d)[:15])),
        ("gemm_lora gate [G, N-8]", lambda m, d: m.gemm_lora(b(16, 16).to(d), b(16, 16).to(d), None, *lo(d),
                                                             gate=f(2, 16).to(d)[:, :8], **gr)),
        ("gemm_lora col_scale bias [N-8]", lambda m, d: m.gemm_lora(b(16, 16).to(d), b(16, 16).to(d), b(16).to(d)[:8], *lo(d),
                                                                    col_scale=f(16).to(d) + 1)),
        ("gemm_fp8 out [M, N-8]", lambda m, d: m.gemm_fp8(e(16, 128).to(d), s8(d)[0], e(16, 128).to(d), s8(d)[1],
                                                          out=b(16, 16).to(d)[:, :8])),
        ("gemm_fp8 residual [M, N-8]", lambda m, d: m.gemm_fp8(e(16, 128).to(d), s8(d)[0], e(16, 128).to(d), s8(d)[1],
                                                               residual=b(16, 16).to(d)[:, :8], epilogue=F_.EPI_BIAS_GATE_RES)),
        ("gemm_fp8 gate rows < groups", lambda m, d: m.gemm_fp8(e(16, 128).to(d), s8(d)[0], e(16, 128).to(d), s8(d)[1],
                                                                gate=f(2, 16).to(d)[:1], **gr)),
        ("gemm_fp8_blocks out [M-1, N]", lambda m, d: m.gemm_fp8_blocks(e(16, 128).to(d), f(16, 1).to(d) + 1, e(16, 128).to(d),
                                                                        s8(d)[1], out=b(16, 16).to(d)[:15])),
        ("gemm_fp8_blocks FP8 GELU bias [N-8]", lambda m, d: m.gemm_fp8_blocks(e(16, 128).to(d), f(16, 1).to(d) + 1, e(128, 128).to(d),
                                                                               f(128).to(d) + 1, b(128).to(d)[:120],
                                                                               epilogue=F_.EPI_BIAS_GELU_TANH_FP8)),
        ("gemm_fp8_blocks mod_index short", lambda m, d: m.gemm_fp8_blocks(e(16, 128).to(d), f(16, 1).to(d) + 1, e(16, 128).to(d),
                                                                           s8(d)[1], gate=f(2, 16).to(d),
                                                                           mod_index=torch.zeros(2, dtype=torch.int32).to(d)[:1], **gr)),
    ]


def osb_ht(m, d, rows, tmap, kinds, H, D):
    return m.HeadTiles(rows, tmap, kinds, H, D, d)


@pytest.mark.parametrize("idx", range(len(_refusals())), ids=[r[0] for r in _refusals()])
def test_refusals(idx):
    import osb200 as osb

    dev = _dev()
    name, call = _refusals()[idx]
    l0 = osb.launch_count()
    with pytest.raises(osb.OsbError):
        call(osb, dev)
    assert osb.launch_count() == l0, "a refused call must launch nothing"
    f0 = F_.launch_count()
    with pytest.raises(F_.OsbError):
        call(F_, "cpu")
    assert F_.launch_count() == f0
    print(f"[conformance] refusal {name}: both raise OsbError")


# ===================================================================================================================
# recorded replay: the double on exactly the arguments the product passes
# ===================================================================================================================
REPLAYED = ("ln_modulate", "gemm", "gemm_lora", "attn_short", "gemm_head_tiles", "attn_tiles", "group_stats", "vae_prep",
            "conv3d", "cfg_euler", "rf_masked_step")


class _Tiles:
    """A HeadTiles argument as recorded: geometry, plus (for attention sources) the decoded kinds at call time."""

    def __init__(self, t, dense=None):
        self.rows, self.map, self.kinds, self.heads, self.head_dim = t.rows, t.map, t.kinds, t.heads, t.head_dim
        self.dense = dense

    def fake(self):
        f = F_.HeadTiles(self.rows, self.map, self.kinds, self.heads, self.head_dim, "cpu")
        if self.dense is not None:
            f.dense.copy_(self.dense)
        return f


class _Recorder:
    """Wraps the real binding's entry points.  Every tensor argument is recorded as a CPU copy of its whole storage plus
    size / stride / offset, one copy per storage per call, so views (qkv[:, :C]) and aliasing (out is residual) survive.
    Calls that route rows to other ranks (scatter / out_scatter) cannot be replayed in one process: counted, skipped."""

    def __init__(self, osb, monkeypatch):
        self.osb, self.calls, self.skipped = osb, [], 0
        for name in REPLAYED:
            monkeypatch.setattr(osb, name, self._wrap(name, getattr(osb, name)))

    def _snap(self, v, stor, sources):
        if isinstance(v, torch.Tensor):
            key = v.untyped_storage().data_ptr()
            if key not in stor:
                raw = torch.empty(0, dtype=torch.uint8, device=v.device).set_(v.untyped_storage())
                stor[key] = raw.cpu()
            return torch.empty(0, dtype=v.dtype).set_(stor[key].untyped_storage(), v.storage_offset(), v.size(), v.stride())
        if isinstance(v, self.osb.HeadTiles):
            dense = torch.stack([read_tiles(v, k).cpu() for k in range(v.kinds)]) if sources else None
            return _Tiles(v, dense)
        if isinstance(v, tuple):
            return tuple(self._snap(t, stor, sources) for t in v)
        return v

    def _wrap(self, name, fn):
        def wrapped(*args, **kw):
            if kw.get("scatter") is not None or kw.get("out_scatter") is not None:
                self.skipped += 1
                return fn(*args, **kw)
            torch.cuda.synchronize()
            stor = {}
            src = name == "attn_tiles"
            rargs = [self._snap(a, stor, src) for a in args]
            rkw = {k: self._snap(v, stor, src) for k, v in kw.items()}
            l0 = self.osb.launch_count()
            r = fn(*args, **kw)
            torch.cuda.synchronize()
            if name == "gemm_head_tiles":
                t = args[3]
                n_kid = args[1].shape[0] // (t.heads * t.head_dim)
                kind0 = kw.get("kind0", 0)
                result = [read_tiles(t, k).cpu() for k in range(kind0, kind0 + n_kid)]
            elif name == "attn_tiles":
                result = args[2].detach().cpu().clone()
            else:
                result = r.detach().cpu().clone()
            self.calls.append((name, rargs, rkw, result, self.osb.launch_count() - l0))
            return r
        return wrapped


def _replay_one(name, args, kw, result):
    """Run one recorded call through the double; returns [(label, got, want, err)] comparisons (err None: exact)."""
    if name == "gemm":
        e = err_gemm(*args, **kw)
        return [("", result, F_.gemm(*args, **kw), e)]
    if name == "gemm_lora":
        a, w, bias, u, b = args
        e = err_gemm(a, w, bias, u=u, b=b, **kw)
        return [("", result, F_.gemm_lora(*args, **kw), e)]
    if name == "ln_modulate":
        e = err_ln(*args, **kw)
        return [("", result, F_.ln_modulate(*args, **kw), e)]
    if name == "attn_short":
        e = err_attn_short(*args, **kw)
        return [("", result, F_.attn_short(*args, **kw), e)]
    if name == "cfg_euler":
        e = err_cfg_euler(*args, **kw)
        return [("", result, F_.cfg_euler(*args, **kw), e)]
    if name == "rf_masked_step":
        e = err_rf_masked_step(*args, **kw)
        return [("", result, F_.rf_masked_step(*args, **kw), e)]
    if name == "conv3d":
        e = err_conv(*args, **kw)
        return [("", result, F_.conv3d(*args, **kw), e)]
    if name == "vae_prep":
        e = None if kw.get("stats") is None and not kw.get("silu") else err_vae_prep(*args, **kw)
        return [("", result, F_.vae_prep(*args, **kw), e)]
    if name == "group_stats":
        full = dict(zip(("x", "groups", "eps"), args), **kw)
        e = err_group_stats(full["x"], full["groups"], full.get("eps", 1e-6))
        want = F_.group_stats(*args, **kw)
        return [(" mean", result[..., 0], want[..., 0], e[..., 0]), (" rstd", result[..., 1], want[..., 1], e[..., 1])]
    if name == "gemm_head_tiles":
        a, w, bias, t = args
        f = t.fake()
        F_.gemm_head_tiles(a, w, bias, f, **kw)
        errs = err_head_tiles(a, w, bias, t.map, t.heads, t.head_dim, **{k: v for k, v in kw.items() if k not in ("kind0", "general")})
        k0 = kw.get("kind0", 0)
        return [(f" kind {k0 + i}", result[i], f.dense[k0 + i], errs[i]) for i in range(len(result))]
    if name == "attn_tiles":
        q, kv, out = args
        fq = q.fake()
        fkv = fq if kv is q else kv.fake()
        qk, kk, vk = kw.get("q_kind", 0), kw.get("k_kind", 1), kw.get("v_kind", 2)
        e = err_attn_tiles(fq.dense[qk], fkv.dense[kk], fkv.dense[vk], fq.map, fkv.map, q.heads, q.head_dim, kw["Lk"],
                           kw["num_seqs"], kv_lens=kw.get("kv_lens"), softmax_scale=kw.get("softmax_scale"),
                           out_map=kw.get("out_map"), out_shape=tuple(out.shape))
        # rows the call does not write keep the recorded content on both sides: E = 0 there, bit-identical
        return [("", result, F_.attn_tiles(fq, fkv, out, **kw), e)]
    raise AssertionError(name)


def _workload(name):
    """One forward of a product path on the GPU (the binding is recorded while it runs)."""
    dev = _dev()
    if name == "stdit3-xs":
        prod, _, cfg = stdit3_pair("xs")
        inp = stdit3_inputs(cfg, 1, 4, 16, 16, device=dev)
        with torch.no_grad():
            prod(**inp)
    elif name.startswith("mmdit"):
        fused, liger = name == "mmdit-fused-flux", name == "mmdit-split-liger"
        m = mmdit_model(fused, liger, device="cuda")
        B, Lt, T, H, W = 2, 40, 3, 6, 8
        g = _gen(3)
        rb = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)  # noqa: E731
        txt_ids, img_ids = mmdit_ids(B, Lt, T, H, W)
        inp = dict(img=rb(B, T * H * W, 64), img_ids=img_ids, txt=rb(B, Lt, 128), txt_ids=txt_ids,
                   timesteps=torch.tensor([0.3, 0.8]), y_vec=rb(B, 96), cond=rb(B, T * H * W, 68),
                   guidance=torch.tensor([4.0, 7.5]))
        with torch.no_grad():
            m(**{k: v.to(dev) for k, v in inp.items()})
    elif name == "vae":
        G = load_golden("vae_blocks.npz")
        m = tiny_vae(G).to(torch.bfloat16).to(dev)
        with torch.no_grad():
            m.encoder(m._to_ndhwc(G["enc_x"].to(torch.bfloat16).to(dev), cpad=8))
            m.decoder(m._to_ndhwc(G["enc_y"][:, :4].to(torch.bfloat16).to(dev)))
    else:
        from opensora.schedulers import RFLOW

        g = torch.Generator(device="cuda").manual_seed(1)
        z = torch.randn(2, 4, 6, 8, 8, device=dev, generator=g).to(torch.bfloat16)
        y = torch.randn(2, 1, 5, 8, device=dev, generator=g)
        fm = torch.tensor([[0.0, 0.5, 1.0, 1.0, 0.3, 1.0], [1.0, 1.0, 0.0, 0.7, 1.0, 1.0]], device=dev)
        RFLOW(num_sampling_steps=2, cfg_scale=6.0).sample(toy_model, z, y, y, frame_mask=fm, generator=g)


@pytest.mark.parametrize("workload", ["stdit3-xs", "mmdit-fused-flux", "mmdit-split-liger", "vae", "rf-masked-loop"])
def test_recorded_replay(workload, monkeypatch):
    import osb200 as osb

    rec = _Recorder(osb, monkeypatch)
    _workload(workload)
    monkeypatch.undo()
    assert rec.calls, "the workload made no binding call"
    stats = {}
    for name, args, kw, result, launches in rec.calls:
        f0 = F_.launch_count()
        for label, got, want, err in _replay_one(name, args, kw, result):
            ratio, same, n = _check(f"replay {workload} {name}{label}", got, want, err, verbose=False,
                                    ulp=ulp_fp32 if name == "group_stats" else ulp_bf16)
            s = stats.setdefault(name + label, [0, 0.0, 0, 0, True])
            s[0] += 1
            s[4] = s[4] and err is None
            s[1], s[2], s[3] = max(s[1], ratio), s[2] + same, s[3] + n
        assert F_.launch_count() - f0 == launches, f"{name}: launch count kernels {launches}, double {F_.launch_count() - f0}"
    for key, (calls, ratio, same, n, exact) in sorted(stats.items()):
        print(f"[conformance] replay {workload} {key}: {calls} calls, {'exact' if exact else 'bound (exact where E = 0)'} "
              f"max|d|/bound={ratio:.3f} bit-identical={same / max(n, 1):.4f} n={n}")
    print(f"[conformance] replay {workload}: {len(rec.calls)} calls replayed, {rec.skipped} scatter calls skipped")
