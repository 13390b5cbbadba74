"""Pins the oracles (CPU, no GPU needed).

* oracle/mmdit_oracle.py against tests/golden/mmdit_blocks.npz — fixtures produced by EXECUTING the
  reference's own MMDiT source (tests/golden/make_golden_mmdit.py; reference files
  opensora/models/mmdit/{layers,math}.py).
* the pieces oracle/stdit3_oracle.py shares with the in-tree MMDiT (RMSNorm cast point, interleaved
  RoPE, LN+modulate, GELU-tanh MLP, exact attention) against the same fixtures.
* STDiT3-specific structure (absent from the reference: PARITY UNPINNED) through properties and a
  self-generated regression fixture (tests/golden/stdit3_xs_selfcheck.npz)."""
import os

import numpy as np
import pytest
import torch

from tests.util import load_golden

from oracle import mmdit_oracle as M
from oracle import stdit3_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
G = load_golden("mmdit_blocks.npz")
C, H, AXES = 64, 2, [8, 12, 12]
TOL = dict(rtol=2e-5, atol=2e-5)


def _w(prefix):
    return {k[len(prefix) + 1:]: v for k, v in G.items() if k.startswith(prefix + ".")}


def test_rmsnorm_matches_reference():
    torch.testing.assert_close(M.rms_norm(G["rms_x"], G["rms_scale"]), G["rms_y"], **TOL)
    # cast point (layers.py:108-111): normalised value is rounded to bf16 BEFORE the weight multiply
    y = M.rms_norm(G["rms_x"].bfloat16(), G["rms_scale"]).float()
    torch.testing.assert_close(y, G["rms_y_bf16"], rtol=0, atol=0)
    n = O.LlamaRMSNorm(G["rms_scale"].numel())
    n.weight.data.copy_(G["rms_scale"])
    torch.testing.assert_close(n(G["rms_x"]), G["rms_y"], **TOL)


def test_rope_and_position_embedding_match_reference():
    pe = M.embed_nd(G["ids"], AXES, 10000)
    torch.testing.assert_close(pe, G["pe_flux"], **TOL)
    torch.testing.assert_close(M.apply_rope(G["rope_q"], pe), G["rope_q_out"], **TOL)
    torch.testing.assert_close(M.apply_rope(G["rope_k"], pe), G["rope_k_out"], **TOL)
    cos, sin = M.liger_embed_nd(G["ids"], AXES, 10000)
    torch.testing.assert_close(cos, G["pe_liger_cos"], **TOL)
    torch.testing.assert_close(sin, G["pe_liger_sin"], **TOL)


def test_stdit3_rotary_is_the_reference_interleaved_rotation():
    """App. A RoPE (single temporal axis) must equal the reference's apply_rope on a 1-axis EmbedND."""
    D, L = 72, 9
    x = torch.randn(2, 3, L, D, generator=torch.Generator().manual_seed(0))
    ids = torch.arange(L, dtype=torch.float32)[None, :, None]
    pe = M.embed_nd(ids, [D], 10000)
    torch.testing.assert_close(O.RotaryEmbedding(D)(x), M.apply_rope(x, pe), **TOL)


def test_timestep_embedding_and_attention_match_reference():
    torch.testing.assert_close(M.timestep_embedding(G["temb_t"], 256), G["temb"], **TOL)
    out = M.attention(G["rope_q"], G["rope_k"], G["attn_v"], G["pe_flux"])
    torch.testing.assert_close(out, G["attn_out_flux"], **TOL)
    # the STDiT3 oracle uses time_factor 1 (upstream v1.2); same construction otherwise
    torch.testing.assert_close(O.timestep_embedding(G["temb_t"] * 1000.0, 256), G["temb"], **TOL)


@pytest.mark.parametrize("tag,fused", [("fused", True), ("split", False)])
def test_double_and_single_blocks_match_reference(tag, fused):
    img, txt, vec, pe = G["img"], G["txt"], G["vec"], G["pe_flux"]
    oi, ot = M.double_stream_block(_w(f"double_{tag}"), img, txt, vec, pe, H, fused)
    torch.testing.assert_close(oi, G[f"double_{tag}_out_img"], **TOL)
    torch.testing.assert_close(ot, G[f"double_{tag}_out_txt"], **TOL)
    o = M.single_stream_block(_w(f"single_{tag}"), torch.cat((txt, img), 1), vec, pe, H, fused)
    torch.testing.assert_close(o, G[f"single_{tag}_out"], **TOL)


def test_last_layer_matches_reference():
    torch.testing.assert_close(M.last_layer(_w("last"), G["img"], G["vec"]), G["last_out"], **TOL)


def test_stdit3_shared_pieces_equal_pinned_mmdit_pieces():
    g = torch.Generator().manual_seed(1)
    x, sh, sc = torch.randn(2, 7, 48, generator=g), torch.randn(2, 1, 48, generator=g), torch.randn(2, 1, 48, generator=g)
    ln = torch.nn.LayerNorm(48, eps=1e-6, elementwise_affine=False)
    torch.testing.assert_close(O.t2i_modulate(ln(x), sh, sc), M.ln_modulate(x, sh, sc), **TOL)
    mlp = O.Mlp(48, 96)
    w = {"0.weight": mlp.fc1.weight, "0.bias": mlp.fc1.bias, "2.weight": mlp.fc2.weight, "2.bias": mlp.fc2.bias}
    torch.testing.assert_close(mlp(x), M._mlp(x, w, ""), **TOL)


# ---- STDiT3 structure: properties (parity unpinned by the reference) ---------------------------------
@pytest.fixture(scope="module")
def xs():
    cfg = O.STDiT3_XS_2_config()
    m = O.STDiT3(cfg).eval()
    O.init_synthetic_weights(m)
    return m, cfg


def test_stdit3_xs_plumbing_config(xs):
    """BASELINE.json configs[0]: STDiT3-XS/2 single denoise step, 1x8x16x16 latent, CPU fp32."""
    m, cfg = xs
    inp = O.synthetic_inputs(cfg, 1, 8, 16, 16)
    with torch.no_grad():
        out = m(**inp)
    assert out.shape == (1, 8, 8, 16, 16) and out.dtype == torch.float32 and torch.isfinite(out).all()
    path = os.path.join(HERE, "golden", "stdit3_xs_selfcheck.npz")
    ref = np.load(path)["out"]
    np.testing.assert_allclose(out.numpy()[:, :, ::2, ::4, ::4], ref, rtol=1e-4, atol=1e-4)


def test_stdit3_text_mask_equals_truncation(xs):
    m, cfg = xs
    inp = O.synthetic_inputs(cfg, 1, 2, 8, 8, lens=[37])
    with torch.no_grad():
        a = m(**inp)
        inp2 = dict(inp)
        y2 = inp["y"].clone()
        y2[:, :, 37:] = 123.0  # masked tokens must not influence the result
        inp2["y"] = y2
        b = m(**inp2)
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)


def test_stdit3_x_mask_all_true_is_identity_and_frames_select(xs):
    m, cfg = xs
    inp = O.synthetic_inputs(cfg, 1, 4, 8, 8)
    with torch.no_grad():
        a = m(**inp)
        b = m(**inp, x_mask=torch.ones(1, 4, dtype=torch.bool))
        c = m(**inp, x_mask=torch.tensor([[False, True, True, True]]))
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)
    assert (a - c).abs().max() > 1e-3


def test_stdit3_batch_independence(xs):
    m, cfg = xs
    inp = O.synthetic_inputs(cfg, 2, 2, 8, 8)
    with torch.no_grad():
        full = m(**inp)
        one = m(**{k: v[1:2] for k, v in inp.items()})
    torch.testing.assert_close(full[1:2], one, rtol=1e-4, atol=1e-4)


def test_algorithmic_flop_model():
    import bench

    assert abs(bench.algorithmic_flops() / 1e12 - 36.13) < 0.01
    # the MMDiT leg's shape and FLOP model: SURVEY.md 8d "MMDiT forward, per sample = 57 (24 C^2 L + 4 L^2 C)": 168.6 TF at 256px
    c = bench.MMDIT_256PX
    C, L = c["hidden_size"], 33 * 12 * 21 + 512
    per_sample = (c["depth"] + c["depth_single_blocks"]) * (24.0 * C * C * L + 4.0 * L * L * C) / 1e12
    assert abs(per_sample - 168.6) < 0.1 and C // c["num_heads"] == sum(c["axes_dim"]) == 128


def test_bench_auxiliary_legs_fail_soft():
    """The extra legs of the bench line report their own failure instead of raising: without a GPU the MMDiT child process
    dies at `cuda.set_device` and the launcher returns the reason; the VAE CPU baseline is a pure host measurement."""
    import bench

    r = bench._vae_cpu_baseline()
    assert "error" not in r and r["value"] > 0 and r["kind"] == "port" and r["unit"] == "frames/s"
    if not torch.cuda.is_available():
        m = bench.mmdit_leg(timeout_s=120)
        assert set(m) == {"error"} and "rc 1" in m["error"]


# ---- causal 3D VAE oracle pinned by reference-executed goldens --------------------------------------
from oracle import vae_oracle as V  # noqa: E402

GV = load_golden("vae_blocks.npz")
VTOL = dict(rtol=1e-4, atol=1e-4)


def _wv(prefix):
    return {k[len(prefix) + 1:]: v for k, v in GV.items() if k.startswith(prefix + ".")}


@pytest.mark.parametrize("tag,stride", [("s111", (1, 1, 1)), ("s122", (1, 2, 2)), ("s222", (2, 2, 2))])
def test_causal_conv3d_matches_reference(tag, stride):
    y = V.causal_conv3d(GV["conv_x"], GV[f"conv_{tag}.w"], GV[f"conv_{tag}.b"], stride)
    torch.testing.assert_close(y, GV[f"conv_{tag}.y"], **VTOL)


def test_causal_conv3d_k1_and_causality():
    torch.testing.assert_close(V.causal_conv3d(GV["conv_x"], GV["conv_k1.w"], GV["conv_k1.b"]), GV["conv_k1.y"], **VTOL)
    x = GV["conv_x"].clone()
    y0 = V.causal_conv3d(x, GV["conv_s111.w"], GV["conv_s111.b"])
    x[:, :, -1] += 1.0  # perturbing the last frame must leave all earlier output frames bit-identical
    y1 = V.causal_conv3d(x, GV["conv_s111.w"], GV["conv_s111.b"])
    assert torch.equal(y0[:, :, :-1], y1[:, :, :-1]) and not torch.equal(y0[:, :, -1], y1[:, :, -1])


@pytest.mark.parametrize("tag,f", [("u222", (2, 2, 2)), ("u122", (1, 2, 2))])
def test_upsample_matches_reference(tag, f):
    y = V.causal_conv3d(V.upsample_causal3d(GV["conv_x"], f), GV[f"up_{tag}.w"], GV[f"up_{tag}.b"])
    torch.testing.assert_close(y, GV[f"up_{tag}.y"], **VTOL)


@pytest.mark.parametrize("tag", ["same", "wide"])
def test_resnet_block_matches_reference(tag):
    torch.testing.assert_close(V.resnet_block(_wv(f"res_{tag}"), "", GV["res_x"], groups=4), GV[f"res_{tag}.y"], **VTOL)


def test_mid_block_and_encoder_decoder_match_reference():
    torch.testing.assert_close(V.mid_block(_wv("mid"), "", GV["res_x"], groups=4), GV["mid.y"], **VTOL)
    down, up = V.stage_plan(4, 4, 8)
    assert down == [(1, 2, 2), (2, 2, 2), (2, 2, 2), None] and up == [(1, 2, 2), (2, 2, 2), (2, 2, 2), None]
    z = V.encoder(_wv("enc"), GV["enc_x"], groups=4, strides=down)
    torch.testing.assert_close(z, GV["enc_y"], rtol=1e-3, atol=1e-3)
    y = V.decoder(_wv("dec"), GV["enc_y"][:, :4], groups=4, factors=up)
    torch.testing.assert_close(y, GV["dec_y"], rtol=1e-3, atol=1e-3)


def test_mmdit_full_model_matches_reference():
    """model.py:154-233 executed by the reference on a tiny config -> pins oracle M.model_forward."""
    cfg = dict(num_heads=H, depth=1, depth_single_blocks=1, axes_dim=AXES, theta=10000, guidance_embed=True,
               cond_embed=True, fused_qkv=True)
    Lt = G["txt"].shape[1]
    out = M.model_forward(_w("model"), cfg, G["model_img"], G["ids"][:, Lt:], G["model_txt"], G["ids"][:, :Lt],
                          G["model_t"], G["model_y"], cond=G["model_cond"], guidance=G["model_g"])
    torch.testing.assert_close(out, G["model_out"], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("tag,sp,tp", [("none", False, False), ("spatial", True, False), ("temporal", False, True), ("both", True, True)])
def test_tiled_autoencoder_matches_reference(tag, sp, tp):
    """autoencoder_kl_causal_3d.py:269-358,384-552 executed by the reference (tests/golden/make_golden_vae_tiled.py)."""
    GT = load_golden("vae_tiled.npz")
    down, up = V.stage_plan(4, 4, 8)
    We, Wd = _wv("enc"), _wv("dec")
    enc_fn = lambda x: V.causal_conv3d(V.encoder(We, x, groups=4, strides=down), GT["quant_w"], GT["quant_b"])  # noqa: E731
    dec_fn = lambda z: V.decoder(Wd, V.causal_conv3d(z, GT["post_w"], GT["post_b"]), groups=4, factors=up)      # noqa: E731
    encode, decode = V.tiled_autoencoder(enc_fn, dec_fn, sample_size=32, sample_tsize=8, spatial=sp, temporal=tp)
    moments = encode(GT["x"])
    z = 0.476986 * moments[:, :4]   # posterior.mode() then scale_factor * (z - shift_factor), :304-311
    torch.testing.assert_close(z, GT[f"z_{tag}"], rtol=1e-3, atol=1e-3)
    y = decode(GT[f"z_{tag}"] / 0.476986)
    torch.testing.assert_close(y, GT[f"y_{tag}"], rtol=2e-3, atol=2e-3)
