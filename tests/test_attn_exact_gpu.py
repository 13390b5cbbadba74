"""The attention kernels bit for bit on the exact cases of tests/exact_attn.py: every output element of `attn_tiles`,
`attn_tiles_fp8`, `attn_short`, `attn_fp8`, `attn_fp8_blocks`, `attn_short_bias` and `attn_frames` must equal the
designed value row (or the exact mean of tied rows), and nothing around the output view may be written.  The cases
place winners in the first, a middle and the last key block, decoys where an off-by-one mask would leak them (past
kv_lens, in the neighbouring packed sequence, in the next frame, at j = i + 1 under a causal mask) and pad key slots that
win for rows whose every visible score is negative, so a masking or indexing bug replaces whole rows."""
import pytest
import torch

from tests import exact_attn as A

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _check(case, got=None):
    import osb200 as osb

    got = case.run(osb) if got is None else got
    torch.cuda.synchronize()
    want = case.want()
    if isinstance(want, tuple):
        (codes, scales), (wc, ws) = got, want
        n_ok = int((codes.view(torch.uint8) == wc.view(torch.uint8)).sum())
        msg = A.first_mismatch(scales, ws) or A.first_mismatch(codes, wc)
        total = codes.numel()
    else:
        same = (got.view(torch.int16) == want.view(torch.int16)) | ((got.float() == 0) & (want.float() == 0))
        n_ok, total = int(same.sum()), same.numel()
        msg = A.first_mismatch(got, want)
    print(f"[exact-attn] {case}: {n_ok} of {total} bit-identical")
    assert msg is None, f"{case}: {msg}"
    assert case.untouched(), f"{case}: wrote outside the output view"


TILE_SELF = [  # (mode, B, T, S, H, D, ties)
    (0, 1, 3, 256, 4, 72, 1), (0, 1, 2, 200, 2, 72, 1), (0, 1, 1, 640, 2, 72, 1), (0, 1, 1, 640, 2, 72, 2),
    (0, 1, 2, 256, 2, 64, 1), (0, 1, 2, 200, 2, 64, 1), (0, 1, 1, 768, 2, 64, 4),   # D 64: 5 stages, 6 key tiles
    (0, 1, 2, 256, 2, 128, 1), (0, 1, 2, 200, 2, 128, 1), (0, 1, 1, 640, 2, 128, 1),
    (1, 2, 16, 12, 2, 72, 1), (1, 1, 17, 10, 2, 72, 1), (1, 1, 64, 8, 4, 72, 1), (1, 1, 100, 6, 2, 72, 1),
    (1, 1, 17, 10, 2, 64, 1), (1, 1, 64, 8, 2, 128, 1),
]


@pytest.mark.parametrize("fp8,mode,B,T,S,H,D,ties", [(False,) + c for c in TILE_SELF]
                         + [(True,) + c for c in TILE_SELF if c[5] != 128])   # FP8 head tiles: head_dim 64 and 72
def test_attn_tiles_self(fp8, mode, B, T, S, H, D, ties):
    case = A.tiles_self_case(mode, B, T, S, H, D, ties=ties, fp8=fp8, seed=hash((mode, T, S, D, ties)) % 1000,
                             device=_dev())
    assert case.winners == ties
    _check(case)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("T,S", [(64, 8), (17, 10)])
def test_attn_tiles_transposed_stream(fp8, T, S):
    """Tiles written from the [B, S, T] stream (contiguous temporal sequences), output rows frame-major (out_map)."""
    case = A.tiles_self_case(1, 1, T, S, 2, 72, transposed=True, fp8=fp8, seed=T, device=_dev())
    _check(case)


def test_attn_tiles_output_scatter():
    """Output rows routed by osb_scatter mode 2 with one rank (the sequence-parallel store path of tile_out_row)."""
    case = A.tiles_self_case(1, 2, 64, 6, 2, 72, scatter=True, seed=5, device=_dev())
    _check(case)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("D", [72, 64])
def test_attn_tiles_cross(fp8, D):
    """kv_lens 300 (every key: pad slots past the third tile), 260 and 7 (decoys just past), 0 (zeros)."""
    case = A.tiles_cross_case(384, 300, [300, 260, 7, 0], 2, D, fp8=fp8, seed=D, device=_dev())
    assert bool((case.expected[3] == 0).all())
    _check(case)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_attn_tiles_more_items_than_ctas(fp8):
    """More work items than 2 x SMs: every persistent CTA walks several items, consecutive sets have different keys,
    so a key tile kept resident for the wrong set changes whole rows."""
    dev = _dev()
    case = A.tiles_self_case(0, 1, 40, 256, 8, 72, fp8=fp8, seed=7, device=dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    assert case.items > 2 * sms, (case.items, sms)
    _check(case)


SHORT = [  # (L, B, T, H, D, kv_lens, ties)
    (1, 2, 1, 4, 128, None, 1), (77, 2, 1, 4, 128, None, 1), (1000, 2, 1, 4, 128, None, 1),
    (1000, 1, 1, 4, 128, None, 2), (2560, 1, 1, 4, 128, None, 1), (333, 2, 1, 4, 128, None, 1),
    (333, 1, 1, 4, 72, None, 1), (333, 1, 1, 4, 64, None, 4),
    (24, 2, 6, 2, 64, [24, 13, 7, 24, 1, 20, 24, 0, 9, 17, 24, 2], 1),
    (40, 1, 3, 2, 72, [40, 31, 5], 1), (300, 2, 1, 2, 72, [300, 260], 1),
]


NORM_ROPE = [  # (L, norm_split, D, rope): MMDiT's joint txt | img sequence with per-stream QK-norm and RoPE
    (1000, 77, 128, "half"), (1000, 77, 128, "interleaved"), (333, 100, 128, "half"), (2560, 512, 128, "half"),
    (200, 77, 72, "interleaved"), (150, 40, 64, "half"), (300, 64, 128, None),
]


@pytest.mark.parametrize("L,split,D,rope", NORM_ROPE)
def test_attn_short_norm_rope(L, split, D, rope):
    """Which RoPE row and which norm weight pair each staged q / k row gets: a wrong position scrambles the code, a key
    staged with the other stream's weight ties with its half-score copy."""
    case = A.short_case(L, 4, D, B=2, norm_split=split, rope=rope, seed=L + split, device=_dev())
    _check(case)


@pytest.mark.parametrize("fn", ["attn_fp8", "attn_fp8_blocks"])
@pytest.mark.parametrize("L,split,rope", [(1000, 77, "half"), (8828, 512, "half"), (333, 100, "interleaved")])
def test_attn_fp8_norm_rope(fn, L, split, rope):
    case = A.short_case(L, 24, 128, B=3, fn=fn, norm_split=split, rope=rope, seed=L, device=_dev())
    _check(case)


@pytest.mark.parametrize("L,B,T,H,D,kv_lens,ties", SHORT)
def test_attn_short(L, B, T, H, D, kv_lens, ties):
    case = A.short_case(L, H, D, B=B, T=T, kv_lens=kv_lens, ties=ties, seed=L + D, device=_dev())
    assert case.winners == (ties if L > 1 else 1)
    _check(case)


@pytest.mark.parametrize("fn", ["attn_fp8", "attn_fp8_blocks"])
@pytest.mark.parametrize("L", [1, 77, 1000, 8828])
def test_attn_fp8(fn, L):
    """MMDiT's FP8 attention, B = 3, H = 24, head_dim 128: pad key slots past L win for the negative rows if leaked.
    The blocks output must be the block rule applied to the exact rows."""
    case = A.short_case(L, 24, 128, B=3, fn=fn, seed=L, device=_dev())
    _check(case)


@pytest.mark.parametrize("variant", ["inf", "finite", "empty"])
def test_attn_short_bias_t5(variant):
    """q = 0, so every score is the bias: head h wins on one relative offset.  -inf elsewhere (key blocks skipped) and
    -300 elsewhere give the same bits; "empty" leaves every row but row 0 of head 0 without a visible key (zeros).
    Heads 1 and 2 sit on the first and the last live relative position of a skipped-or-not key block."""
    case = A.t5_bias_case(300, 400, 4, B=2, variant=variant, seed=11, device=_dev())
    assert case.offsets[1:3].tolist() == [1, 63]
    _check(case)


def test_attn_short_bias_causal():
    """CLIP's causal mask: decoys at j = i + 1."""
    case = A.causal_case(77, 4, B=2, seed=12, device=_dev())
    assert len(case.decoys) > 0
    _check(case)


FRAMES = [  # (hw, q_frames, q_frame0, k_frames, batch)
    (4, 40, 0, None, 1), (64, 6, 0, None, 1), (100, 5, 0, None, 1), (1000, 3, 0, None, 1),
    (100, 2, 2, 5, 1), (1000, 2, 1, 4, 1), (64, 4, 0, None, 2), (100, 3, 1, 5, 2),
]


@pytest.mark.parametrize("hw,q_frames,q_frame0,k_frames,batch", FRAMES)
def test_attn_frames(hw, q_frames, q_frame0, k_frames, batch):
    case = A.frames_case(hw, q_frames, q_frame0=q_frame0, k_frames=k_frames, batch=batch, seed=hw + q_frame0,
                         device=_dev())
    _check(case)
