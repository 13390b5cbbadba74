"""The FP8 (e4m3) MLP path on the CPU: the stand-in entries of tests/fake_osb200.py against the contract arithmetic
of tests/fp8_ref.py on its edge cases, the host-side STDiT3 with `enable_fp8()` against the FP8-emulating oracle,
`disable_fp8()`, the K % 128 refusal and the ctypes mirror of `osb_gemm_fp8_args`."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from tests import fp8_ref as R
from tests.models import stdit3_inputs, stdit3_pair
from tests.util import rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn


def _rows(seed=0, rows=12, K=256):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, K, generator=g) * torch.logspace(-3, 2, rows)[:, None]
    x[2] = 0.0                                    # all-zero row: scale 1, codes 0
    x[5, 7] = -1000.0                             # the row's amax lands on -448
    x[6] = 3.0                                    # constant row: every code is exactly 448
    return x


def test_quant_rows_matches_the_contract(fake_osb):
    x = _rows().to(torch.bfloat16)
    q, s = fake_osb.quant_rows_fp8(x)
    rq, rs = R.quantize(x.float())
    assert q.dtype == E4M3 and s.dtype == torch.float32
    assert torch.equal(s, rs) and torch.equal(q.double(), rq)
    assert s[2] == 1.0 and not q[2].float().any()
    assert q[5, 7].float() == -448.0 and torch.all(q[6].float() == 448.0)
    # a strided view (row stride > K) quantizes its K columns only
    wide = torch.randn(12, 384).to(torch.bfloat16)
    q2, s2 = fake_osb.quant_rows_fp8(wide[:, :256])
    rq2, rs2 = R.quantize(wide[:, :256].float())
    assert torch.equal(s2, rs2) and torch.equal(q2.double(), rq2)
    with pytest.raises(fake_osb.OsbError):
        fake_osb.quant_rows_fp8(torch.zeros(4, 12, dtype=torch.bfloat16))   # K % 8


def test_ln_modulate_fp8_quantizes_the_fp32_value(fake_osb):
    """The fc1 input is the fp32 LN+modulate row, quantized without a bf16 rounding first; mod_index selects the table."""
    g = torch.Generator().manual_seed(1)
    rows, C = 16, 256
    x = (torch.randn(rows, C, generator=g) * 3).to(torch.bfloat16)
    x[4] = 0.0                                    # LN of a constant row is 0: modulate leaves the shift only
    mod = torch.randn(3, 2, C, generator=g)
    mod_index = torch.tensor([2, 0, 1, 2], dtype=torch.int32)
    q, s = fake_osb.ln_modulate_fp8(x, mod[:, 0], mod[:, 1], group_rows=4, mod_index=mod_index)
    xf = x.float()
    gi = mod_index.long()[torch.arange(rows) // 4]
    y = F.layer_norm(xf, (C,), eps=1e-6) * (1 + mod[gi, 1]) + mod[gi, 0]
    rq, rs = R.quantize(y)
    assert torch.allclose(s, rs, rtol=1e-6, atol=0)
    step = (rq.abs() * 2.0 ** -3).clamp(min=2.0 ** -9)           # one e4m3 step at the value
    assert ((q.double() - rq).abs() <= step).all()
    assert (q.double() == rq).float().mean() > 0.99
    # quantizing the bf16-rounded row instead would differ on a visible share of the codes
    qb, _ = R.quantize(y.to(torch.bfloat16).float())
    assert not torch.equal(qb, rq)
    with pytest.raises(fake_osb.OsbError):
        fake_osb.ln_modulate_fp8(torch.zeros(2, 8192, dtype=torch.bfloat16), mod[:1, 0].repeat(1, 32)[:, :8192],
                             mod[:1, 1].repeat(1, 32)[:, :8192], group_rows=2)


@pytest.mark.parametrize("epilogue", [0, 1, 2])
def test_gemm_fp8_matches_dequantized_fp32(fake_osb, epilogue):
    g = torch.Generator().manual_seed(2)
    M, N, K = 70, 48, 384
    a = _rows(3, M, K)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    a8, sa = R.quantize(a)
    w8, sw = R.quantize(w)
    bias = torch.randn(N, generator=g).to(torch.bfloat16)
    res = torch.randn(M, N, generator=g).to(torch.bfloat16)
    gate = torch.randn(4, N, generator=g)
    mod_index = torch.tensor([3, 1, 0, 2, 1], dtype=torch.int32)
    kw = dict(residual=res, gate=gate, group_rows=16, mod_index=mod_index) if epilogue == 2 else {}
    a_view = torch.zeros(M, K + 128, dtype=E4M3)
    a_view[:, :K] = a8.float().to(E4M3)
    got = fake_osb.gemm_fp8(a_view[:, :K], sa, w8.float().to(E4M3), sw, bias, epilogue=epilogue, **kw)
    ref = R.dequantize(a8, sa).double() @ R.dequantize(w8, sw).double().t() + bias.double()
    if epilogue == 1:
        ref = F.gelu(ref, approximate="tanh")
    elif epilogue == 2:
        gi = mod_index.long()[torch.arange(M) // 16]
        ref = ref * gate[gi].double() + res.double()
    assert got.dtype == torch.bfloat16
    assert rel_l2(got, ref) < 3e-3
    for bad in (dict(K=288), dict(epilogue=3)):
        Kb = bad.get("K", K)
        with pytest.raises(fake_osb.OsbError):
            fake_osb.gemm_fp8(torch.zeros(8, Kb, dtype=E4M3), torch.ones(8), torch.zeros(8, Kb, dtype=E4M3), torch.ones(8),
                          epilogue=bad.get("epilogue", 0))


def test_host_stdit3_fp8_follows_the_emulation(fake_osb):
    """XS/2 at hidden 256 with FP8 MLPs on the stand-in, against the fp32 oracle.  The yardstick is the FP8-emulation
    reference: the oracle in bf16 with its block MLPs at the FP8 rounding points (tests/fp8_ref.py), measured in the same
    test.  The product may not be more than 1.1x further from the fp32 oracle than that reference, plain and with an
    x_mask (the mod_index route)."""
    prod, oracle, cfg = stdit3_pair("xs64", device="cpu")
    prod.enable_fp8()
    inp = stdit3_inputs(cfg, 2, 4, 8, 8, lens=[cfg.model_max_length, 9])
    xm = torch.ones(2, 4, dtype=torch.bool)
    xm[1, 1:3] = False
    ob = stdit3_pair("xs64", device="cpu")[1].to(torch.bfloat16)
    for kw in ({}, {"x_mask": xm}):
        fake_osb.reset()
        with torch.no_grad():
            ref = oracle(**inp, **kw)
            out = prod(**inp, **kw)
            with R.fp8_mlps(ob):
                emu = ob(**inp, **kw).float()
            floor = ob(**inp, **kw).float()
        r_emu, r_out, r_bf = rel_l2(emu, ref), rel_l2(out, ref), rel_l2(floor, ref)
        print(f"[fp8 host] {'x_mask' if kw else 'plain'}: product {r_out:.3e}, FP8 emulation {r_emu:.3e}, "
              f"bf16 oracle {r_bf:.3e} (rel-L2 against the fp32 oracle)")
        assert r_out < 1.1 * r_emu and r_emu > r_bf, (r_out, r_emu, r_bf)
        names = [c[0] for c in fake_osb.calls]
        nb = 2 * cfg.depth
        assert names.count("gemm_fp8") == 2 * nb and names.count("ln_modulate_fp8") == nb
        # the fc2 input once per block; on the CPU the weights (2 per block) are quantized by the first forward
        assert names.count("quant_rows_fp8") == nb + (2 * nb if not kw else 0)
        assert names.count("ln_modulate") == nb + 1


def test_disable_fp8_restores_the_bf16_path(fake_osb):
    prod, _, cfg = stdit3_pair("xs64", device="cpu")
    inp = stdit3_inputs(cfg, 1, 4, 8, 8)
    with torch.no_grad():
        before = prod(**inp)
        prod.enable_fp8()
        fp8 = prod(**inp)
        prod.disable_fp8()
        fake_osb.reset()
        after = prod(**inp)
    assert not torch.equal(before, fp8)
    assert torch.equal(before, after)
    assert not any(k[0] == "fp8" for k in prod._cache)
    assert not any(c[0].endswith("fp8") for c in fake_osb.calls)


def test_fp8_refuses_hidden_sizes_off_the_k_block(fake_osb):
    """XS/2 as shipped has hidden size 288, not a multiple of the 128-element e4m3 k-block."""
    from opensora.models.stdit.stdit3 import STDiT3_XS_2

    m = STDiT3_XS_2().to(torch.bfloat16)
    with pytest.raises(ValueError, match="multiples of 128"):
        m.enable_fp8()
    assert m._fp8 is False


def test_fp8_refuses_sizes_beyond_the_kernels():
    """The FP8 LN+modulate holds rows of at most 4096 columns, the row quantizer at most 8192: wider models are refused
    by enable_fp8() instead of failing at their first forward.  (Meta tensors: only the shapes exist.)"""
    from opensora.models.stdit.stdit3 import STDiT3, STDiT3Config

    for hidden, ratio in ((4224, 1.0), (2176, 4.0)):   # C > 4096; MLP width 8704 > 8192
        with torch.device("meta"):
            m = STDiT3(STDiT3Config(depth=1, hidden_size=hidden, num_heads=hidden // 64, mlp_ratio=ratio,
                                    caption_channels=128, model_max_length=8))
        with pytest.raises(ValueError, match="<= 4096"):
            m.enable_fp8()
        assert m._fp8 is False


def test_gemm_fp8_args_layout_matches_header():
    import subprocess
    import tempfile

    import osb200

    fields = [
        ("sizeof(osb_gemm_fp8_args)", ctypes.sizeof(osb200.GemmFp8Args)),
        ("offsetof(osb_gemm_fp8_args, a_scale)", osb200.GemmFp8Args.a_scale.offset),
        ("offsetof(osb_gemm_fp8_args, mod_index)", osb200.GemmFp8Args.mod_index.offset),
        ("offsetof(osb_gemm_fp8_args, M)", osb200.GemmFp8Args.M.offset),
        ("offsetof(osb_gemm_fp8_args, gate_stride)", osb200.GemmFp8Args.gate_stride.offset),
        ("offsetof(osb_gemm_fp8_args, epilogue)", osb200.GemmFp8Args.epilogue.offset),
        ("offsetof(osb_gemm_fp8_args, block_n)", osb200.GemmFp8Args.block_n.offset),
    ]
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "probe.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "osb200.h"\nint main(){\n')
            for expr, _ in fields:
                f.write(f'printf("%zu\\n", (size_t)({expr}));\n')
            f.write("return 0;}\n")
        exe = os.path.join(d, "probe")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    for (expr, mine), theirs in zip(fields, got):
        assert mine == theirs, (expr, mine, theirs)
