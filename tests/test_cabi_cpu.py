"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/osb200.h declares, and the product path refuses to run without a GPU (no fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "osb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(osb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import osb200

    declared = _header_symbols()
    assert declared, "no entry points parsed from include/osb200.h"
    lib = ctypes.CDLL(osb200.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), f"libosb200.so does not export {name}"
    assert sorted(osb200.EXPORTS) == declared


def test_version_and_error_string_without_gpu():
    import osb200

    assert osb200.version() >= 100
    assert isinstance(osb200.last_error(), str)
    assert osb200.launch_count() >= 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_ops_fail_loudly_without_gpu():
    import osb200

    with pytest.raises(osb200.OsbError):
        osb200.init()
    a = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(osb200.OsbError):
        osb200.gemm(a, a)
    # calling the C entry point directly before osb_init must return an error code, not crash
    args = osb200.GemmArgs()
    rc = osb200._lib.osb_gemm_bf16(ctypes.byref(args), None)
    assert rc != 0 and "osb_init" in osb200.last_error()


def test_ctypes_struct_layout_matches_header():
    """sizeof of the ctypes mirrors must equal the C structs (checked against a gcc-compiled probe)."""
    import subprocess
    import tempfile

    import osb200

    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "probe.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "osb200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n",'
                    "sizeof(osb_gemm_args), sizeof(osb_attn_short_args), offsetof(osb_gemm_args, epilogue),"
                    "offsetof(osb_attn_short_args, softmax_scale), sizeof(osb_conv3d_args), sizeof(osb_vae_prep_args),"
                    "offsetof(osb_conv3d_args, block_n), offsetof(osb_vae_prep_args, cp));return 0;}\n")
        exe = os.path.join(d, "probe")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert ctypes.sizeof(osb200.GemmArgs) == sizes[0]
    assert ctypes.sizeof(osb200.AttnShortArgs) == sizes[1]
    assert osb200.GemmArgs.epilogue.offset == sizes[2]
    assert osb200.AttnShortArgs.softmax_scale.offset == sizes[3]
    assert ctypes.sizeof(osb200.Conv3dArgs) == sizes[4]
    assert ctypes.sizeof(osb200.VaePrepArgs) == sizes[5]
    assert osb200.Conv3dArgs.block_n.offset == sizes[6]
    assert osb200.VaePrepArgs.cp.offset == sizes[7]


def test_registry_and_state_dict_contract():
    from opensora.registry import MODELS, build_module
    from oracle.stdit3_oracle import STDiT3 as Oracle, STDiT3_XS_2_config

    m = build_module(dict(type="STDiT3-XS/2"), MODELS)
    o = Oracle(STDiT3_XS_2_config())
    a, b = m.state_dict(), o.state_dict()
    assert set(a) == set(b)
    assert all(a[k].shape == b[k].shape for k in a)
    assert "STDiT3-XL/2" in MODELS and "STDiT3-3B/2" in MODELS
    xl = build_module(dict(type="STDiT3-XL/2", depth=1), MODELS)  # kwargs override like the reference's factories
    assert xl.hidden_size == 1152 and xl.num_heads == 16 and xl.depth == 1
    assert build_module(m, MODELS) is m and build_module(None, MODELS) is None
    with pytest.raises(TypeError):
        build_module(3, MODELS)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_model_forward_has_no_cpu_fallback():
    import osb200
    from opensora.models.stdit.stdit3 import STDiT3_XS_2

    m = STDiT3_XS_2()
    with pytest.raises(osb200.OsbError):
        m(torch.zeros(1, 4, 2, 4, 4), torch.zeros(1), torch.zeros(1, 1, 300, 4096), fps=torch.ones(1),
          height=torch.ones(1), width=torch.ones(1))


def test_product_tree_knows_nothing_of_the_test_double_or_the_oracle():
    """tests/fake_osb200.py (host-logic stand-in) and oracle/ are test infrastructure: no file of the shipped package may
    reference either, so there is no path by which the product could route around the CUDA library."""
    import os

    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open-sora_b200")
    offenders = []
    for d, _, files in os.walk(root):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(d, f), errors="ignore").read()
                if "fake_osb200" in txt or "import oracle" in txt or "from oracle" in txt:
                    offenders.append(os.path.join(d, f))
    assert not offenders, offenders


def test_head_tile_and_exchange_struct_layouts_match_header():
    """ctypes mirrors of the round-2 structs (head tiles, peer-memory exchange) against a gcc-compiled probe: sizes and the
    offsets of the last / alignment-sensitive fields."""
    import subprocess
    import tempfile

    import osb200

    fields = [
        ("sizeof(osb_tile_map)", ctypes.sizeof(osb200.TileMap)),
        ("sizeof(osb_head_tiles_args)", ctypes.sizeof(osb200.HeadTilesArgs)),
        ("offsetof(osb_head_tiles_args, norm_w)", osb200.HeadTilesArgs.norm_w.offset),
        ("offsetof(osb_head_tiles_args, rope_sin)", osb200.HeadTilesArgs.rope_sin.offset),
        ("sizeof(osb_attn_tiles_args)", ctypes.sizeof(osb200.AttnTilesArgs)),
        ("offsetof(osb_attn_tiles_args, num_seqs)", osb200.AttnTilesArgs.num_seqs.offset),
        ("offsetof(osb_attn_tiles_args, out_scatter)", osb200.AttnTilesArgs.out_scatter.offset),
        ("sizeof(osb_scatter)", ctypes.sizeof(osb200.Scatter)),
        ("offsetof(osb_scatter, peer)", osb200.Scatter.peer.offset),
        ("sizeof(osb_comm_barrier_args)", ctypes.sizeof(osb200.CommBarrierArgs)),
        ("offsetof(osb_comm_barrier_args, flags_peer)", osb200.CommBarrierArgs.flags_peer.offset),
        ("OSB_MAX_PEERS", osb200.MAX_PEERS),
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


def test_tile_map_arithmetic():
    """tile_map() (host) against the documented rules of include/osb200.h: packing, ragged tiles, balanced key tiles."""
    import osb200

    def km(*a, **k):
        return osb200.tile_map(*a, **k).key()

    assert km(0, 256) == (0, 256, 0, 0, 1, 2, 128)                  # STDiT3 spatial: 2 tiles per sequence
    assert km(1, 64, 256, 64) == (1, 64, 256, 64, 2, 1, 128)        # temporal: 2 sequences per tile
    assert km(0, 300, keys_only=True) == (0, 300, 0, 0, 1, 3, 128)  # T5 keys: 128 + 128 + 44
    assert km(0, 16384, pack=False) == (0, 16384, 0, 0, 1, 128, 128)
    assert km(0, 64, pack=False) == (0, 64, 0, 0, 1, 1, 64)         # cross-attention queries are never packed
    assert km(1, 17, 100, 17) == (1, 17, 100, 17, 7, 1, 128)        # 7 x 17 = 119 rows -> 128
    assert km(1, 100, 6, 100) == (1, 100, 6, 100, 1, 1, 112)
    m = osb200.tile_map(0, 200)
    assert osb200._lib.osb_head_tiles_per_head(ctypes.byref(m), 5 * 200) == 10
    m = osb200.tile_map(1, 16, 12, 16)
    assert osb200._lib.osb_head_tiles_per_head(ctypes.byref(m), 2 * 16 * 12) == 3   # 24 sequences, 8 per tile


def test_stand_in_tile_map_is_the_binding():
    """tests/fake_osb200.py uses the binding's own `tile_map` (host arithmetic, no device), so the host tests tile every
    sequence exactly as the kernels do.  The arithmetic itself is checked against the rules of include/osb200.h for every
    mode, L in 1..400, keys_only and pack."""
    import osb200
    from tests import fake_osb200

    assert fake_osb200.tile_map is osb200.tile_map and fake_osb200.TileMap is osb200.TileMap
    for mode in (0, 1):
        for L in range(1, 401):
            for kw in ({}, {"keys_only": True}, {"pack": False}, {"keys_only": True, "pack": False}):
                S, T = (12, L) if mode == 1 else (0, 0)
                m = fake_osb200.tile_map(mode, L, S, T, **kw)
                assert m.key()[:4] == (mode, L, S, T)
                assert 16 <= m.tile_rows <= 128 and m.tile_rows % 16 == 0, (mode, L, kw, m.key())
                if L <= 64 and kw.get("pack", True) and not kw.get("keys_only", False):
                    assert m.G == 128 // L and m.tps == 1 and m.G * L <= m.tile_rows < m.G * L + 16, (mode, L, kw, m.key())
                else:
                    assert m.G == 1 and m.tps == -(-L // m.tile_rows) and (L > 128) == (m.tile_rows == 128 and m.tps > 1)
                    assert m.tile_rows * (m.tps - 1) < L <= m.tile_rows * m.tps, (mode, L, kw, m.key())
                rows = 3 * L * (S if mode == 1 else 1)
                seqs = rows // L
                want = -(-seqs // m.G) if m.G > 1 else seqs * m.tps
                assert osb200._lib.osb_head_tiles_per_head(ctypes.byref(m), rows) == want
