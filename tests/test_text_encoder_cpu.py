"""text_embedder (T5 v1.1 / CLIP text encoders on osb200) without a GPU: the fp32 oracle and the bucket table against
goldens produced by executing the reference's own HFEmbedder (tests/golden/make_golden_text.py), the host model on the
binding stand-in, checkpoint and config refusals, the reference's padding rules, the registry / prepare_models path of
the reference's inference configs, and the sampler's `prepare` / `prepare_api` fed by the new embedders."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import text_fixtures as tf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "text_encoders.npz")


def _golden():
    return np.load(GOLDEN)


def _t5_dir(tmp_path, cfg=None, weights=None, fmt="safetensors", name="google/t5-v1_1-xxl"):
    cfg = cfg or tf.T5_TINY
    return tf.write_checkpoint(str(tmp_path / name), cfg, weights if weights is not None else tf.t5_weights(cfg, tf.SEED_T5), fmt)


def _clip_dir(tmp_path, cfg=None, weights=None, fmt="safetensors", name="openai/clip-vit-large-patch14"):
    cfg = cfg or tf.CLIP_TINY
    return tf.write_checkpoint(str(tmp_path / name), cfg, weights if weights is not None else tf.clip_weights(cfg, tf.SEED_CLIP), fmt)


def _rel(a, b):
    a, b = torch.as_tensor(a).float(), torch.as_tensor(b).float()
    return float((a - b).norm() / b.norm())


def _within_floor(out, golden, floor_out):
    """The bf16 model may miss the fp32 golden by what the oracle run in bf16 (the reference's rounding points, the same
    bf16 weights) misses it by, with a 25% + 2e-3 margin for the different rounding points of fused epilogues."""
    err, floor = _rel(out, golden), _rel(floor_out, golden)
    assert err <= 1.25 * floor + 2e-3, (err, floor)


def _t5_floor(ids):
    from oracle import text_oracle as O

    return O.t5_encode(tf.t5_weights(tf.T5_TINY, tf.SEED_T5), tf.T5_TINY, ids, dtype=torch.bfloat16)


# ---- oracle and bucket table ----------------------------------------------------------------------------------------
def test_oracle_matches_reference_goldens():
    from oracle import text_oracle as O

    g = _golden()
    w = tf.t5_weights(tf.T5_TINY, tf.SEED_T5)
    for key in ("t5", "t5_pad"):
        out = O.t5_encode(w, tf.T5_TINY, torch.from_numpy(g[f"{key}_ids"]))
        np.testing.assert_allclose(out.numpy(), g[f"{key}_out"], rtol=2e-5, atol=2e-5)
    for tag in ("legacy", "eos"):
        cfg = json.loads(str(g[f"clip_{tag}_cfg"]))
        out = O.clip_encode(tf.clip_weights(cfg, tf.SEED_CLIP), cfg, torch.from_numpy(g[f"clip_{tag}_ids"]))
        np.testing.assert_allclose(out.numpy(), g[f"clip_{tag}_out"], rtol=2e-5, atol=2e-5)
    # the two pooling rules pick different rows on these prompts
    ids = torch.from_numpy(g["clip_eos_ids"])
    assert not torch.equal(O.clip_pool_index(ids, 300), O.clip_pool_index(ids, 2))


def test_bucket_table_matches_transformers():
    from opensora.models.text.conditioner import relative_position_bucket
    from oracle.text_oracle import t5_bucket

    g = _golden()
    rel = torch.arange(-1023, 1024)
    np.testing.assert_array_equal(relative_position_bucket(rel, 32, 128).numpy(), g["t5_buckets"])
    np.testing.assert_array_equal(t5_bucket(rel, 32, 128).numpy(), g["t5_buckets"])


# ---- host model on the stand-in ---------------------------------------------------------------------------------------
def test_t5_host_model_on_stand_in_vs_golden(fake_osb, tmp_path):
    from opensora.models.text.conditioner import HFEmbedder

    g = _golden()
    emb = HFEmbedder(_t5_dir(tmp_path), max_length=512, tokenizer=tf.t5_tokenizer(), torch_dtype=torch.bfloat16)
    text = [str(t) for t in g["t5_text"]]
    assert torch.equal(emb.tokenize(text), torch.from_numpy(g["t5_ids"]))
    out = emb(text)
    assert out.shape == (2, 512, 128) and out.dtype == torch.bfloat16
    _within_floor(out, g["t5_out"], _t5_floor(torch.from_numpy(g["t5_ids"])))
    # one q|k|v GEMM, the bias attention, o + residual, two RMSNorms, gated GELU, wo + residual per layer; final norm
    names = [c[0] for c in fake_osb.calls]
    assert names.count("rms_norm") == 2 * 2 + 1 and names.count("attn_short") == 2 and names.count("gemm") == 4 * 2
    # the padding of the reference: added_tokens + L made a multiple of seq_align with pad_token_id
    ids = emb.tokenize(text, added_tokens=5, seq_align=16)
    assert torch.equal(ids, torch.from_numpy(g["t5_pad_ids"])) and (5 + ids.shape[1]) % 16 == 0
    _within_floor(emb(text, added_tokens=5, seq_align=16), g["t5_pad_out"], _t5_floor(ids))


@pytest.mark.parametrize("tag", ["legacy", "eos"])
def test_clip_host_model_on_stand_in_vs_golden(fake_osb, tmp_path, tag):
    from opensora.models.text.conditioner import HFEmbedder

    g = _golden()
    cfg = json.loads(str(g[f"clip_{tag}_cfg"]))
    emb = HFEmbedder(_clip_dir(tmp_path, cfg), max_length=77, torch_dtype=torch.bfloat16)
    ids = torch.from_numpy(g[f"clip_{tag}_ids"])
    out = emb.encode(ids)
    assert out.shape == (3, 128)
    from oracle import text_oracle as O

    _within_floor(out, g[f"clip_{tag}_out"], O.clip_encode(tf.clip_weights(cfg, tf.SEED_CLIP), cfg, ids, dtype=torch.bfloat16))


@pytest.mark.parametrize("fmt", ["sharded", "bin"])
def test_checkpoint_formats(fake_osb, tmp_path, fmt):
    from opensora.models.text.conditioner import HFEmbedder

    g = _golden()
    emb = HFEmbedder(_t5_dir(tmp_path, fmt=fmt), max_length=512, tokenizer=tf.t5_tokenizer())
    ids = torch.from_numpy(g["t5_ids"])
    _within_floor(emb.encode(ids), g["t5_out"], _t5_floor(ids))


def test_full_checkpoints_keep_only_the_text_encoder(fake_osb, tmp_path):
    """A T5ForConditionalGeneration checkpoint (decoder, LM head, tied embed_tokens) and a CLIPModel checkpoint (vision
    tower, projections, position_ids, text_config nesting) load; the extra tensors are not read."""
    from opensora.models.text.conditioner import HFEmbedder

    w = tf.t5_weights(tf.T5_TINY, tf.SEED_T5)
    w.update({"decoder.block.0.layer.0.SelfAttention.q.weight": torch.zeros(128, 128), "lm_head.weight": torch.zeros(8, 128),
              "encoder.embed_tokens.weight": w["shared.weight"].clone()})
    HFEmbedder(_t5_dir(tmp_path, weights=w), max_length=16, tokenizer=tf.t5_tokenizer())
    cw = tf.clip_weights(tf.CLIP_TINY, tf.SEED_CLIP)
    cw.update({"vision_model.embeddings.class_embedding": torch.zeros(8), "text_projection.weight": torch.zeros(8, 128),
               "logit_scale": torch.zeros(()), "text_model.embeddings.position_ids": torch.arange(77)[None]})
    HFEmbedder(_clip_dir(tmp_path, {"text_config": tf.CLIP_TINY, "model_type": "clip"}, weights=cw), max_length=77)


# ---- refusals -----------------------------------------------------------------------------------------------------
def test_key_refusals_name_the_key(fake_osb, tmp_path):
    from opensora.models.text.conditioner import HFEmbedder

    base = tf.t5_weights(tf.T5_TINY, tf.SEED_T5)
    k = "encoder.block.1.layer.1.DenseReluDense.wi_1.weight"
    cases = {
        "missing": ({kk: v for kk, v in base.items() if kk != k}, k),
        "unexpected": (dict(base, **{"encoder.block.1.layer.0.SelfAttention.relative_attention_bias.weight": torch.zeros(32, 2)}),
                       "encoder.block.1.layer.0.SelfAttention.relative_attention_bias.weight"),
        "shape": (dict(base, **{k: torch.zeros(320, 64)}), k),
    }
    for i, (w, key) in enumerate(cases.values()):
        with pytest.raises(RuntimeError, match=key.replace(".", r"\.")):
            HFEmbedder(_t5_dir(tmp_path, weights=w, name=f"t5-{i}"), max_length=16, tokenizer=tf.t5_tokenizer())
    cw = tf.clip_weights(tf.CLIP_TINY, tf.SEED_CLIP)
    ck = "text_model.encoder.layers.0.mlp.fc1.bias"
    with pytest.raises(RuntimeError, match=ck.replace(".", r"\.")):
        HFEmbedder(_clip_dir(tmp_path, weights={kk: v for kk, v in cw.items() if kk != ck}), max_length=77)


@pytest.mark.parametrize("case", ["t5_relu", "t5_gated_relu", "t5_dkv", "clip_gelu", "clip_head"])
def test_config_refusals(fake_osb, tmp_path, case):
    from opensora.models.text.conditioner import HFEmbedder

    cfg, is_clip, match = {
        "t5_relu": (dict(tf.T5_TINY, feed_forward_proj="relu"), False, "relu"),
        "t5_gated_relu": (dict(tf.T5_TINY, feed_forward_proj="gated-relu"), False, "gated-relu"),
        "t5_dkv": (dict(tf.T5_TINY, d_kv=32, num_heads=4), False, "d_kv = 32"),
        "clip_gelu": (dict(tf.CLIP_TINY, hidden_act="gelu"), True, "gelu"),
        "clip_head": (dict(tf.CLIP_TINY, num_attention_heads=4), True, "head size 32"),
    }[case]
    d = tf.write_checkpoint(str(tmp_path / ("openai/x" if is_clip else "t5")), cfg, {})
    with pytest.raises(fake_osb.OsbError, match=match):
        HFEmbedder(d, max_length=16, tokenizer=tf.t5_tokenizer())


def test_dtype_and_device_refusals(fake_osb, tmp_path):
    from opensora.models.text.conditioner import HFEmbedder

    with pytest.raises(fake_osb.OsbError, match="bfloat16"):
        HFEmbedder(_t5_dir(tmp_path), max_length=16, torch_dtype=torch.float32, tokenizer=tf.t5_tokenizer())
    emb = HFEmbedder(_t5_dir(tmp_path), max_length=16, tokenizer=tf.t5_tokenizer())
    with pytest.raises(fake_osb.OsbError, match="input_ids on"):
        emb.encode(torch.zeros(1, 16, dtype=torch.long, device="meta"))


def test_forward_has_no_cpu_fallback(tmp_path):
    """With the real binding (no GPU here) a CPU model refuses to run instead of computing in eager torch."""
    try:
        import osb200
    except Exception:   # the library is not built: that is a refusal too
        pytest.skip("libosb200.so is not built")
    from opensora.models.text.conditioner import HFEmbedder

    emb = HFEmbedder(_t5_dir(tmp_path), max_length=16, tokenizer=tf.t5_tokenizer())
    with pytest.raises(osb200.OsbError):
        emb(["1 2 3"])


def test_clip_layernorm_weight_range(fake_osb, tmp_path):
    """osb_ln_modulate multiplies by 1 + (w - 1): exact for bf16 w == 0 or 2^-16 <= |w| < 2^16, refused outside."""
    from opensora.models.text.conditioner import HFEmbedder, clip_ln_scale

    top = torch.tensor(2.0 ** 16).bfloat16().float() - 2.0 ** 8   # largest bf16 below 2^16
    ok = torch.tensor([0.0, 2.0 ** -16, -(2.0 ** -16), float(top), -float(top), 1.0, 0.37]).bfloat16()
    s = clip_ln_scale(ok, "t")
    assert torch.equal(1.0 + s[0], ok.float())
    for bad in (2.0 ** -17, 2.0 ** 16, -(2.0 ** 16)):
        with pytest.raises(fake_osb.OsbError, match="layer_norm2"):
            clip_ln_scale(torch.tensor([1.0, bad]).bfloat16(), "text_model.encoder.layers.1.layer_norm2")
    cw = tf.clip_weights(tf.CLIP_TINY, tf.SEED_CLIP)
    cw["text_model.encoder.layers.1.layer_norm2.weight"][3] = 2.0 ** 17
    with pytest.raises(fake_osb.OsbError, match=r"text_model\.encoder\.layers\.1\.layer_norm2"):
        HFEmbedder(_clip_dir(tmp_path, weights=cw), max_length=77)


# ---- registry, prepare_models, prepare / prepare_api ------------------------------------------------------------
def _reference_text_cfgs(tmp_path):
    """The t5 / clip dicts of the reference's configs/diffusion/inference/256px.py, with the checkpoint paths pointing at
    seeded toy checkpoints under the same directory names."""
    t5 = dict(type="text_embedder", from_pretrained=_t5_dir(tmp_path), max_length=512, shardformer=True)
    clip = dict(type="text_embedder", from_pretrained=_clip_dir(tmp_path), max_length=77)
    return t5, clip


def test_reference_config_dicts_build_through_the_registry(fake_osb, tmp_path, monkeypatch):
    from opensora.models.text import conditioner
    from opensora.registry import MODELS, build_module

    monkeypatch.setattr(conditioner.HFEmbedder, "tokenizer", property(lambda self: tf.clip_tokenizer() if self.is_clip else tf.t5_tokenizer()))
    t5_cfg, clip_cfg = _reference_text_cfgs(tmp_path)
    t5 = build_module(t5_cfg, MODELS, device_map="cpu", torch_dtype=torch.bfloat16)
    clip = build_module(clip_cfg, MODELS, device_map="cpu", torch_dtype=torch.bfloat16)
    assert isinstance(t5, conditioner.HFEmbedder) and not t5.is_clip and t5.output_key == "last_hidden_state"
    assert clip.is_clip and clip.output_key == "pooler_output" and clip.max_length == 77
    assert t5(["5 6 7"]).shape == (1, 512, 128) and clip(["5 6 7"]).shape == (1, 128)
    with pytest.raises(AssertionError, match="Shardformer"):
        build_module(dict(clip_cfg, shardformer=True), MODELS)


def test_prepare_models_on_a_toy_config(fake_osb, tmp_path, monkeypatch):
    from opensora.models.text import conditioner
    from opensora.utils import sampling as S
    from tests import sampling_toys as T

    monkeypatch.setattr(conditioner.HFEmbedder, "tokenizer", property(lambda self: tf.clip_tokenizer() if self.is_clip else tf.t5_tokenizer()))
    t5_cfg, clip_cfg = _reference_text_cfgs(tmp_path)
    model, ae = T.ToyDenoiser(), T.ToyAE(causal=True)
    cfg = dict(model=model, ae=ae, t5=t5_cfg, clip=clip_cfg)
    m, a, t5, clip, opt = S.prepare_models(cfg, "cpu", torch.bfloat16)
    assert m is model and a is ae and opt == {} and isinstance(t5, conditioner.HFEmbedder) and clip.is_clip
    with pytest.raises(KeyError, match="autoencoder_2d"):
        S.prepare_models(dict(cfg, img_flux=dict(type="flux"), img_flux_ae=dict(type="autoencoder_2d")), "cpu", torch.bfloat16)


def test_prepare_and_prepare_api_fed_by_the_embedders(fake_osb, tmp_path):
    from opensora.models.text.conditioner import HFEmbedder
    from opensora.utils import sampling as S
    from tests import sampling_toys as T

    t5 = HFEmbedder(_t5_dir(tmp_path), max_length=32, tokenizer=tf.t5_tokenizer())
    clip = HFEmbedder(_clip_dir(tmp_path), max_length=77, tokenizer=tf.clip_tokenizer())
    img = torch.randn(2, 16, 1, 8, 8, dtype=torch.bfloat16)
    inp = S.prepare(t5, clip, img, ["4 5 6", "7 8"], seq_align=8)
    L = inp["txt"].shape[1]
    assert (L + inp["img"].shape[1]) % 8 == 0 and L >= 32
    assert torch.equal(inp["txt"][1], t5(["7 8"], added_tokens=inp["img"].shape[1], seq_align=8)[0])
    assert torch.equal(inp["y_vec"], clip(["4 5 6", "7 8"]))
    # the text-to-video toy scenario of prepare_api, with the real embedders in place of the toy ones
    model = T.ToyDenoiser().to(torch.bfloat16)
    ae = T.ToyAE(causal=True).to(torch.bfloat16)
    api = S.prepare_api(model, ae, t5, clip, {})
    opt = S.sanitize_sampling_option(S.SamplingOption(height=32, width=48, num_frames=17, num_steps=3, guidance=7.5,
                                                      guidance_img=3.0, temporal_reduction=4, is_causal_vae=True, seed=3))
    x = api(opt, cond_type="t2v", text=["3 4 5", "9"], neg=["10", "11 12"])
    assert x.shape == (2, 3, 17, 32, 48) and torch.isfinite(x.float()).all()
    assert len(model.seen) == 3
    names = [c[0] for c in fake_osb.calls]
    assert names.count("cfg_euler") == 3 and names.count("attn_short") > 0


def test_enum_values_match_header(tmp_path):
    """The new epilogue values of the ctypes binding against a gcc-compiled probe of include/osb200.h."""
    src, exe = str(tmp_path / "p.c"), str(tmp_path / "p")
    with open(src, "w") as fh:
        fh.write('#include <stdio.h>\n#include "osb200.h"\nint main(void){printf("%d %d\\n", OSB_EPI_GATED_GELU, '
                 'OSB_EPI_BIAS_QUICK_GELU);return 0;}\n')
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
    vals = [int(v) for v in subprocess.check_output([exe], text=True).split()]
    from tests import fake_osb200

    assert vals == [3, 4] == [fake_osb200.EPI_GATED_GELU, fake_osb200.EPI_BIAS_QUICK_GELU]
    text = open(os.path.join(ROOT, "open-sora_b200", "osb200", "__init__.py")).read()
    assert "EPI_GATED_GELU, EPI_BIAS_QUICK_GELU = 3, 4" in text
