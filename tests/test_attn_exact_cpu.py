"""The exact attention cases of tests/exact_attn.py on the CPU: every builder passes its own budget at reduced sizes, a
dense fp64 softmax over the built operands gives the expected rows, cases that break the construction are refused, a
mask off by one changes the result (the cases can see the bugs they target), and every CPU stand-in of the attention
entry points reproduces the expected rows bit for bit."""
import math

import pytest
import torch

from tests import exact_attn as A

# (id, builder, kwargs, leak): reduced sizes of the GPU matrix; `leak` is the off-by-one mask the case is built to catch
CASES = [
    ("tiles-spatial-200-72", A.tiles_self_case, dict(mode=0, B=1, T=2, S=200, H=2, D=72), "limit"),
    ("tiles-spatial-640-64-ties", A.tiles_self_case, dict(mode=0, B=1, T=1, S=640, H=2, D=64, ties=2), "limit"),
    ("tiles-temporal-16-128", A.tiles_self_case, dict(mode=1, B=1, T=16, S=10, H=2, D=128), "next_seq"),
    ("tiles-temporal-17-72", A.tiles_self_case, dict(mode=1, B=1, T=17, S=9, H=2, D=72), "next_seq"),
    ("tiles-temporal-100-transposed", A.tiles_self_case, dict(mode=1, B=1, T=100, S=3, H=2, D=72, transposed=True),
     "limit"),
    ("tiles-cross", A.tiles_cross_case, dict(N=128, Ly=300, lens=[260, 7, 0, 300], H=2, D=72), "limit"),
    ("tiles_fp8-temporal-64", A.tiles_self_case, dict(mode=1, B=1, T=64, S=4, H=2, D=64, fp8=True), "next_seq"),
    ("tiles_fp8-cross", A.tiles_cross_case, dict(N=128, Ly=300, lens=[260, 7, 0], H=2, D=72, fp8=True), "limit"),
    ("short-77-128", A.short_case, dict(L=77, H=2, D=128), "limit"),
    ("short-333-72-ties", A.short_case, dict(L=333, H=2, D=72, ties=4), "limit"),
    ("short-packed-kv", A.short_case, dict(L=24, H=2, D=64, B=2, T=3, kv_lens=[24, 13, 7, 24, 1, 20]), "limit"),
    ("short-norm-rope-interleaved", A.short_case, dict(L=200, H=2, D=72, norm_split=77, rope="interleaved"),
     "rope_shift"),
    ("short-norm-rope-half-split", A.short_case, dict(L=333, H=2, D=128, norm_split=77, rope="half"), "split"),
    ("short-norm-64-split", A.short_case, dict(L=150, H=2, D=64, norm_split=40, rope="half"), "split"),
    ("fp8-norm-rope", A.short_case, dict(L=200, H=2, D=128, B=2, fn="attn_fp8", norm_split=77, rope="interleaved"),
     "rope_shift"),
    ("fp8-1", A.short_case, dict(L=1, H=2, D=128, B=3, fn="attn_fp8"), "limit"),
    ("fp8-200", A.short_case, dict(L=200, H=2, D=128, B=2, fn="attn_fp8"), "limit"),
    ("fp8_blocks-200", A.short_case, dict(L=200, H=2, D=128, B=2, fn="attn_fp8_blocks"), "limit"),
    ("bias-t5-inf", A.t5_bias_case, dict(Lq=140, Lk=150, H=2, variant="inf"), None),
    ("bias-t5-finite", A.t5_bias_case, dict(Lq=140, Lk=150, H=2, variant="finite"), None),
    ("bias-t5-empty", A.t5_bias_case, dict(Lq=140, Lk=150, H=2, variant="empty"), None),
    ("bias-causal", A.causal_case, dict(L=77, H=2), "limit"),
    ("frames-4", A.frames_case, dict(hw=4, q_frames=5), "limit"),
    ("frames-100-q0", A.frames_case, dict(hw=100, q_frames=2, q_frame0=1, k_frames=4, batch=2), "limit"),
]
IDS = [c[0] for c in CASES]


def _build(i):
    _, builder, kw, _ = CASES[i]
    return builder(seed=i, **kw)


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_budget_and_dense_reference(i):
    case = _build(i)
    assert case.winners in ((2,) if "ties=2" in case.name else (4,) if "ties=4" in case.name else (0, 1)), case.winners
    ref = A.reference(case)
    assert float((ref - case.expected).abs().max()) <= A.REF_TOL, case
    if case.kv_lens is not None:   # rows of an empty key set are zero
        for s in (case.kv_lens == 0).nonzero().flatten().tolist():
            assert bool((case.expected[s] == 0).all())


@pytest.mark.parametrize("i", [i for i, c in enumerate(CASES) if c[3]], ids=[c[0] for c in CASES if c[3]])
def test_off_by_one_mask_changes_the_output(i):
    case = _build(i)
    wrong = A.reference(case, leak=CASES[i][3]).to(torch.bfloat16)
    right = case.expected.to(torch.bfloat16)
    changed = (wrong != right).any(-1)
    assert bool(changed.any()), f"{case}: a mask off by one leaves every row unchanged"
    print(f"[exact-attn] {case}: off-by-one mask ({CASES[i][3]}) changes {int(changed.sum())} of {changed.numel()} rows")


def test_t5_variants_expect_the_same_rows():
    """-inf elsewhere (key blocks skipped) and a finite -300 elsewhere must give the same bits."""
    a = A.t5_bias_case(140, 150, 2, variant="inf", seed=3)
    b = A.t5_bias_case(140, 150, 2, variant="finite", seed=3)
    assert torch.equal(a.expected, b.expected)
    e = A.t5_bias_case(140, 150, 2, variant="empty", seed=3)
    assert bool((e.expected[:, 0, 1:] == 0).all()) and bool((e.expected[:, 0, 0] != 0).any())


def test_rejects_a_shrunk_margin():
    case = A.short_case(L=77, H=2, D=72, seed=1)
    case.scale /= 4                       # the winner's 2 alpha lead over any other code falls to 87 log2 units
    with pytest.raises(A.BudgetError, match="beats another visible key"):
        A.check_budget(case)


def test_rejects_a_visible_decoy():
    case = A.tiles_cross_case(N=128, Ly=300, lens=[260, 7], H=2, D=72, seed=2)
    case.kv_lens = case.kv_lens + 1       # the first decoy of each sample becomes visible
    with pytest.raises(A.BudgetError):
        A.check_budget(case)
    causal = A.causal_case(L=40, H=2, seed=2)
    causal.bias = causal.bias.clone()
    causal.bias[causal.Lq] = 0.0          # key i + 1 visible to row i
    with pytest.raises(A.BudgetError):
        A.check_budget(causal)


def test_rejects_inexact_operands():
    case = A.short_case(L=77, H=2, D=64, seed=4)
    case.v = case.v.clone()
    case.v[0, 0, 0, 0] = 1.125           # four significant bits
    with pytest.raises(A.BudgetError, match="every value"):
        A.check_budget(case)
    case = A.short_case(L=77, H=2, D=64, seed=4)
    case.q = case.q * 1.5                 # q / alpha no longer integral
    with pytest.raises(A.BudgetError, match="integers"):
        A.check_budget(case)


def test_rejects_a_three_way_tie():
    case = A.short_case(L=77, H=2, D=64, ties=2, seed=5)
    case.k = case.k.clone()
    s, keys = case.tie_keys[0]
    spare = next(j for j in range(case.Lk) if j not in keys.tolist())
    case.k[s, :, spare] = case.k[s, :, keys[0]]
    case.v = case.v.clone()
    case.v[s, :, spare] = case.v[s, :, keys[0]]
    with pytest.raises(A.BudgetError):
        A.check_budget(case)


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_cpu_double_gives_the_expected_bits(fake_osb, i):
    case = _build(i)
    got = case.run(fake_osb)
    want = case.want()
    if isinstance(want, tuple):
        (codes, scales), (wc, ws) = got, want
        A.assert_bits(f"{case} scales", scales, ws)
        A.assert_bits(f"{case} codes", codes, wc)
    else:
        A.assert_bits(str(case), got, want)
    assert case.untouched(), f"{case}: wrote outside the output view"


def test_value_scales_vary_by_head_channel_and_block():
    """FP8 value scales (amax per scale group) differ between heads, channels and 128-key blocks, so a value read with
    the wrong scale is off by a power of two."""
    case = A.short_case(L=1000, H=4, D=128, B=3, fn="attn_fp8", seed=9)
    seq_amax = case.v.abs().amax(2)                              # [nseq, H, D]: attn_fp8's groups
    assert len(torch.unique(seq_amax)) >= 4
    blk = torch.nn.functional.pad(case.v.abs(), (0, 0, 0, 24)).view(3, 4, 8, 128, 128).amax(3)
    assert bool((blk != blk[:, :, :1]).any())                    # attn_tiles_fp8's groups (128-key tiles)
    m, _ = torch.frexp(blk)
    assert bool((m == 0.875).all())                              # every group's amax is 1.75 x 2^E


def test_packed_decoys_follow_the_query_tile():
    """attn_short packs 128 // L sequences per query tile across batch elements: decoys cross batch boundaries too."""
    case = A.short_case(L=24, H=2, D=64, B=2, T=3, seed=1)
    sq, sk = case.decoys[:, 0], case.decoys[:, 2]
    assert bool(((sq // 3) != (sk // 3)).any()) and bool(((sq // 5) == (sk // 5)).all())


def test_alpha_budget():
    """The per-head_dim alpha gives a margin of >= 160 log2 units and a negative winner within 2^10."""
    for D, a in A.ALPHA.items():
        unit = a * D ** -0.5 * A.LOG2E
        assert A.MARGIN <= unit and 5 * unit <= A.WIN_MAX, (D, unit)
        assert A.n_codes(D) - A.FILLERS >= 1000
    assert math.isclose(A.LOG2E, 1 / math.log(2))
