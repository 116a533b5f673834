"""CPU-side checks of the C ABI: the library loads and exports every symbol include/avc_b200.h declares;
the size / offset queries (host-only functions) agree with the reference's state-dict layout."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "avc_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(avc_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    from avatarclip_b200 import _lib
    L = _lib.lib()
    syms = _declared_symbols()
    assert len(syms) >= 8
    for s in syms:
        assert hasattr(L, s), s
    assert L.avc_abi_version() == 3
    assert L.avc_build_arch() == b"sm_90a"


def test_param_layout_matches_reference_state_dict():
    import avatarclip_b200 as ab
    from avatarclip_b200._lib import NeusCfg, lib, check
    state = torch.load(os.path.join(ROOT, "tests", "golden", "neus_small.pt"), map_location="cpu", weights_only=False)
    sdf = ab.SDFNetwork(**state["sdf_kw"])
    col = ab.RenderingNetwork(**state["col_kw"])
    sdf.load_state_dict(state["sdf_state"])                  # shipped checkpoint keys / shapes
    col.load_state_dict(state["col_state"], strict=False)    # (no extra_lin in the file: main.py:617)
    assert list(sdf.state_dict().keys())[:3] == ["lin0.bias", "lin0.weight_g", "lin0.weight_v"]
    cfg = NeusCfg(sdf_d_in=3, sdf_d_out=129, sdf_d_hidden=128, sdf_n_layers=3, sdf_skip_mask=1 << 3, sdf_multires=6,
                  sdf_scale=1.0, col_d_feature=128, col_d_hidden=128, col_n_layers=1, n_samples=32, n_importance=32,
                  up_sample_steps=4, engine=0)
    n = C.c_int64()
    check(lib().avc_neus_param_count(C.byref(cfg), C.byref(n)), "count")
    want = sum(p.numel() for p in sdf.parameters()) + sum(p.numel() for p in col.parameters()) + 1
    assert n.value == want
    sz = C.c_size_t()
    check(lib().avc_neus_workspace_bytes(C.byref(cfg), 512, C.byref(sz)), "ws")
    assert sz.value > 0
    bad = NeusCfg(sdf_d_in=2)
    assert lib().avc_neus_param_count(C.byref(bad), C.byref(n)) == -1     # AVC_E_BADCFG


def test_no_cpu_fallback():
    import avatarclip_b200 as ab
    sdf = ab.SDFNetwork(3, 33, 32, 2, skip_in=(), multires=6)
    col = ab.RenderingNetwork(32, "no_view_dir", 6, 3, 32, 1, extra_color=True)
    var = ab.SingleVarianceNetwork(0.3)
    ren = ab.NeuSRenderer(None, sdf, var, col, 8, 8, 0, 2, 0.0, extra_color=True)
    o = torch.zeros(4, 3)
    with pytest.raises(ab.AvcError):
        ren.render(o, o, torch.zeros(4, 1), torch.ones(4, 1))
