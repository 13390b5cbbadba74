"""text_embedder kernels and encoders on the H100: osb_attn_short_bias (T5 relative bias and the -inf causal mask),
osb_rms_norm and the gated-GELU / quick-GELU GEMM epilogues against fp32 restatements, with the CPU stand-in's entries
(tests/fake_osb200_text.py) held to the same element-wise bounds; whole-encoder parity against the oracle at the golden
configs, full T5-XXL and full CLIP-L; CUDA-graph replay.  Each case prints max |delta| / bound."""
import json
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _osb():
    import osb200

    osb200.init()
    return osb200


def _ulp(x):
    """bf16 ulp of |x| (spacing above the value's binade)."""
    a = x.abs().float().clamp_min(2.0 ** -126)
    return torch.pow(2.0, torch.floor(torch.log2(a)) - 7)


def _check(name, k, d, bound):
    k, d = k.float(), d.float()
    assert torch.isfinite(k).all(), name
    r = float(((k - d).abs() / bound).max())
    same = float((k == d).float().mean())
    print(f"{name}: max |k-d|/bound {r:.3f}, bit-identical {same:.4f}")
    assert r <= 1.0, (name, r)


# ---- bias attention ---------------------------------------------------------------------------------------------
def _attn_case(L, H, kind, B, kv_lens=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = 64
    qkv = (torch.randn(B * L, 3 * H * D, generator=g, device="cuda") * (0.125 if kind == "t5" else 1.0)).bfloat16()
    rel = torch.arange(-(L - 1), L, device="cuda")
    if kind == "t5":
        from opensora.models.text.conditioner import relative_position_bucket

        table = torch.randn(32, H, generator=g, device="cuda").bfloat16().float()
        bias = table[relative_position_bucket(rel.cpu(), 32, 128).cuda()].t().contiguous()
        scale = 1.0
    else:
        bias = torch.where(rel > 0, float("-inf"), 0.0).float().contiguous()
        scale = D ** -0.5
    lens = torch.randint(1, L + 1, (B,), generator=g, device="cuda").int() if kv_lens else None
    return qkv, bias, scale, lens


def _attn_ref(qkv, bias, scale, lens, B, L, H):
    """fp32 restatement with the kernel's rounding of the unnormalised P; also (P|V|) per output element."""
    D = 64
    q, k, v = (qkv[:, i * H * D:(i + 1) * H * D].float().view(B, L, H, D).transpose(1, 2) for i in range(3))
    rel = torch.arange(L, device="cuda")[None, :] - torch.arange(L, device="cuda")[:, None] + L - 1
    s = q @ k.transpose(-1, -2) * scale + bias.view(-1, 2 * L - 1)[:, rel][None]
    if lens is not None:
        s = s.masked_fill((torch.arange(L, device="cuda")[None, :] >= lens[:, None].long())[:, None, None, :], float("-inf"))
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    o = (p.bfloat16().float() @ v) / l
    pv = (p / l) @ v.abs()
    return (o.transpose(1, 2).reshape(B * L, H * D), pv.transpose(1, 2).reshape(B * L, H * D))


ATTN_CASES = [(L, kind) for L in (1, 7, 77, 128, 300, 512, 513) for kind in ("t5", "causal")]


@pytest.mark.parametrize("L,kind", ATTN_CASES)
@pytest.mark.parametrize("kv_lens", [False, True])
def test_attn_short_bias(L, kind, kv_lens):
    osb = _osb()
    from tests import fake_osb200_text as fake

    H, B = 4, 3
    qkv, bias, scale, lens = _attn_case(L, H, kind, B, kv_lens, seed=L)
    C = H * 64
    kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H, head_dim=64,
              kv_lens=lens, softmax_scale=scale)
    out = torch.zeros(B * L, C, dtype=torch.bfloat16, device="cuda")
    osb.attn_short_bias(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, bias, **kw)
    d = torch.zeros_like(out)
    n0 = fake.launch_count()
    fake.attn_short_bias(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], d, bias, **kw)
    assert fake.launch_count() == n0 + 1
    ref, pv = _attn_ref(qkv, bias, scale, lens, B, L, H)
    # P rounded to bf16 (2^-8 relative) in both, plus fp32 exp / sum terms (2^-10), plus the output rounding
    bound = _ulp(ref) + 2.0 ** -7 * pv + 1e-6
    _check(f"attn_short_bias L={L} {kind} kv_lens={kv_lens} kernel-ref", out, ref, bound)
    _check(f"attn_short_bias L={L} {kind} kv_lens={kv_lens} kernel-stand-in", out, d, bound + _ulp(d))


def test_attn_short_bias_packed_sequences():
    """Lq < 64: 128 // L sequences share a query tile (block-diagonal keys), with the relative bias per sequence."""
    osb = _osb()
    from tests import fake_osb200_text as fake

    for L, kind in ((7, "t5"), (16, "causal"), (33, "t5")):
        H, B = 2, 11
        qkv, bias, scale, _ = _attn_case(L, H, kind, B, seed=100 + L)
        C = H * 64
        kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
                  head_dim=64, softmax_scale=scale)
        out = torch.zeros(B * L, C, dtype=torch.bfloat16, device="cuda")
        osb.attn_short_bias(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], out, bias, **kw)
        d = fake.attn_short_bias(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], torch.zeros_like(out), bias, **kw)
        ref, pv = _attn_ref(qkv, bias, scale, None, B, L, H)
        bound = _ulp(ref) + 2.0 ** -7 * pv + 1e-6
        _check(f"attn_short_bias packed L={L} {kind}", out, ref, bound)
        _check(f"attn_short_bias packed L={L} {kind} stand-in", out, d, bound + _ulp(d))


def test_attn_short_bias_refusals():
    osb = _osb()
    from tests import fake_osb200_text as fake

    q = torch.zeros(8, 3 * 72, dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(15, device="cuda")
    for impl in (osb, fake):
        n0 = impl.launch_count()
        with pytest.raises(impl.OsbError):   # head_dim 72 is not built for the bias variant
            impl.attn_short_bias(q[:, :72], q[:, 72:144], q[:, 144:], torch.zeros(8, 72, dtype=torch.bfloat16, device="cuda"),
                                 bias, num_seqs=1, seqs_per_batch=1, q_strides=(8, 0, 1), k_strides=(8, 0, 1), Lq=8, Lk=8,
                                 num_heads=1, head_dim=72)
        with pytest.raises(impl.OsbError):   # wrong bias length
            impl.attn_short_bias(q[:, :64], q[:, 64:128], q[:, 128:192], torch.zeros(8, 64, dtype=torch.bfloat16, device="cuda"),
                                 torch.zeros(14, device="cuda"), num_seqs=1, seqs_per_batch=1, q_strides=(8, 0, 1),
                                 k_strides=(8, 0, 1), Lq=8, Lk=8, num_heads=1, head_dim=64)
        assert impl.launch_count() == n0


# ---- RMSNorm --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [8, 64, 128, 760, 4096])
def test_rms_norm(C):
    osb = _osb()
    from tests import fake_osb200_text as fake

    g = torch.Generator(device="cuda").manual_seed(C)
    x = (torch.randn(333, C, generator=g, device="cuda") * 3).bfloat16()
    w = (1 + 0.3 * torch.randn(C, generator=g, device="cuda")).bfloat16()
    k = osb.rms_norm(x, w, eps=1e-6)
    d = fake.rms_norm(x, w, eps=1e-6)
    # restated roundings; rsqrtf and the fp32 sum order may move the first rounding by one ulp, then w * that ulp
    t_ulp = _ulp(d.float() / w.float().clamp_min(1e-30))
    bound = _ulp(d) + w.float().abs() * t_ulp
    _check(f"rms_norm C={C}", k, d, bound)
    same = float((k == d).float().mean())
    assert same > 0.99, same


def test_rms_norm_refusals():
    osb = _osb()
    from tests import fake_osb200_text as fake

    for impl in (osb, fake):
        n0 = impl.launch_count()
        for C in (12, 4104):
            with pytest.raises(impl.OsbError):
                impl.rms_norm(torch.zeros(4, C, dtype=torch.bfloat16, device="cuda"), torch.ones(C, dtype=torch.bfloat16, device="cuda"))
        assert impl.launch_count() == n0


# ---- GEMM epilogues ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("block_n", [64, 128, 192, 256])
@pytest.mark.parametrize("N", [64, 208, 1024, 2064])   # ragged against every block_n; the gated output N / 2 keeps ldd % 8 == 0
@pytest.mark.parametrize("epi", ["gated", "quick"])
def test_text_epilogues(block_n, N, epi):
    osb = _osb()
    from tests import fake_osb200_text as fake

    g = torch.Generator(device="cuda").manual_seed(N + block_n)
    M, K = 300, 392
    a = torch.randn(M, K, generator=g, device="cuda").bfloat16()
    w = (torch.randn(N, K, generator=g, device="cuda") * K ** -0.5).bfloat16()
    bias = None if epi == "gated" else (0.1 * torch.randn(N, generator=g, device="cuda")).bfloat16()
    e = osb.EPI_GATED_GELU if epi == "gated" else osb.EPI_BIAS_QUICK_GELU
    k = osb.gemm(a, w, bias, epilogue=e, block_n=block_n)
    n0 = fake.launch_count()
    d = fake.gemm(a, w, bias, epilogue=e, block_n=block_n)
    assert fake.launch_count() == n0 + 1 and k.shape == d.shape == (M, N // 2 if epi == "gated" else N)
    acc = a.double() @ w.double().t() + (0 if bias is None else bias.double())
    mag = a.double().abs() @ w.double().abs().t()
    gam = K * 2.0 ** -24 / (1 - K * 2.0 ** -24) * mag   # Higham gamma_K on the fp32 dot products
    if epi == "gated":
        x0, x1 = acc[:, 0::2], acc[:, 1::2]
        ref = (0.5 * x0 * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x0 + 0.044715 * x0 ** 3)))) * x1
        # d/dx gelu <= 1.13; tanh.approx.f32 has 2^-10.99 relative error: 0.5 |x0| |x1| 2^-10.99
        E = 1.13 * gam[:, 0::2] * x1.abs() + (x0.abs() + gam[:, 0::2]) * 1.13 * gam[:, 1::2] + 0.5 * x0.abs() * x1.abs() * 2.0 ** -10.99
    else:
        ref = acc * torch.sigmoid(1.702 * acc)
        E = 1.13 * gam + acc.abs() * 2.0 ** -20   # __expf and the division: a few fp32 ulps of the sigmoid
    bound = (_ulp(ref) + E + 1e-30).float()
    _check(f"gemm {epi} N={N} block_n={block_n} kernel-fp64", k, ref.float(), bound)
    _check(f"gemm {epi} N={N} block_n={block_n} kernel-stand-in", k, d, bound + _ulp(d) + E.float())


# ---- whole encoders -------------------------------------------------------------------------------------------------
def _encoder_parity(name, out, fp32, bf16, cap):
    err = float((out.float() - fp32).norm() / fp32.norm())
    floor = float((bf16.float() - fp32).norm() / fp32.norm())
    print(f"{name}: rel-L2 error {err:.3e}, bf16 floor {floor:.3e}, ratio {err / floor:.3f}")
    assert err <= 1.1 * floor and err < cap, (name, err, floor)


def test_golden_config_encoders_vs_oracle(tmp_path):
    _osb()
    from oracle import text_oracle as O
    from tests import text_fixtures as tf
    from opensora.models.text.conditioner import HFEmbedder

    g = np.load(os.path.join(ROOT, "tests", "golden", "text_encoders.npz"))
    w = tf.t5_weights(tf.T5_TINY, tf.SEED_T5)
    wb = {k_: v.bfloat16().float() for k_, v in w.items()}   # identical bf16 weights for model and oracle
    emb = HFEmbedder(tf.write_checkpoint(str(tmp_path / "t5"), tf.T5_TINY, wb), max_length=512, device_map="cuda",
                     torch_dtype=torch.bfloat16, tokenizer=tf.t5_tokenizer())
    ids = torch.from_numpy(g["t5_ids"]).cuda()
    _encoder_parity("T5 tiny", emb.encode(ids), O.t5_encode(wb, tf.T5_TINY, ids), O.t5_encode(wb, tf.T5_TINY, ids, torch.bfloat16), 5e-2)
    for tag in ("legacy", "eos"):
        cfg = json.loads(str(g[f"clip_{tag}_cfg"]))
        wc = {k_: v.bfloat16().float() for k_, v in tf.clip_weights(cfg, tf.SEED_CLIP).items()}
        emb = HFEmbedder(tf.write_checkpoint(str(tmp_path / "openai" / tag), cfg, wc), max_length=77, device_map="cuda",
                         torch_dtype=torch.bfloat16)
        ids = torch.from_numpy(g[f"clip_{tag}_ids"]).cuda()
        _encoder_parity(f"CLIP tiny {tag}", emb.encode(ids), O.clip_encode(wc, cfg, ids),
                        O.clip_encode(wc, cfg, ids, torch.bfloat16), 5e-2)


def test_full_t5_xxl_vs_oracle(tmp_path):
    _osb()
    from oracle import text_oracle as O
    from tests import text_fixtures as tf, text_gpu_common as G
    from opensora.models.text.conditioner import _t5_shapes

    cfg = tf.T5_XXL
    w = G.device_weights(_t5_shapes(cfg), False, 5, cfg["d_model"])
    emb = G.build(str(tmp_path), cfg, w, False, 512)
    gen = torch.Generator(device="cuda").manual_seed(9)
    ids = torch.randint(2, cfg["vocab_size"], (2, 512), generator=gen, device="cuda")
    ids[0, 300:] = 0   # pads attend and are attended, as with attention_mask=None
    out = emb.encode(ids)
    torch.backends.cuda.matmul.allow_tf32 = False
    # random 24-layer T5 weights grow the residual stream: the bf16 floor itself is about 0.11 here
    _encoder_parity("T5-XXL 2x512", out, O.t5_encode(w, cfg, ids), O.t5_encode(w, cfg, ids, torch.bfloat16), 0.15)


def test_full_clip_l_vs_oracle_and_graph_replay(tmp_path):
    _osb()
    from oracle import text_oracle as O
    from tests import text_fixtures as tf, text_gpu_common as G
    from opensora.models.text.conditioner import _clip_shapes

    cfg = tf.CLIP_L
    w = G.device_weights(_clip_shapes(cfg), True, 6, cfg["hidden_size"])
    emb = G.build(str(tmp_path), cfg, w, True, 77)
    gen = torch.Generator(device="cuda").manual_seed(10)
    ids = torch.randint(1, cfg["vocab_size"] - 2, (2, 77), generator=gen, device="cuda")
    ids[:, 0] = cfg["bos_token_id"]
    ids[0, 20] = ids[1, 50] = cfg["vocab_size"] - 1   # eos; the legacy rule pools at the largest id
    ids[0, 21:] = ids[1, 51:] = cfg["vocab_size"] - 1
    out = emb.encode(ids)
    torch.backends.cuda.matmul.allow_tf32 = False
    _encoder_parity("CLIP-L 2x77", out, O.clip_encode(w, cfg, ids), O.clip_encode(w, cfg, ids, torch.bfloat16), 5e-2)
    # graph replay of the same encode equals the eager call, bit for bit
    static = ids.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        emb.encode(static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        res = emb.encode(static)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(res, out)


def test_t5_graph_replay_equals_eager(tmp_path):
    _osb()
    from tests import text_fixtures as tf, text_gpu_common as G
    from opensora.models.text.conditioner import _t5_shapes

    cfg = dict(tf.T5_TINY, num_layers=3)
    emb = G.build(str(tmp_path), cfg, G.device_weights(_t5_shapes(cfg), False, 3, cfg["d_model"]), False, 300)
    ids = torch.randint(0, cfg["vocab_size"], (2, 300), device="cuda")
    eager = emb.encode(ids)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        emb.encode(ids)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        res = emb.encode(ids)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(res, eager)
