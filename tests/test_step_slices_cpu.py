"""The per-slice gradient bars of tests/test_step_at_scale_gpu.py catch defects that the flat rel-L2 < 1e-3 of the older step
tests cannot see.  The fp64 oracle step is the reference and the fp32 oracle step plays the product, on the benchmark's
networks, weights, text and canvas at 64 rays, under comparison (a)'s definition (the CLIP cotangent held fixed) and the
benchmark's (a) bars.  The fp32 oracle passes; each planted defect fails on the slice it touches."""
import pytest
import torch

import bench
import util_neus as U
import util_step as S
from oracle import neus
from oracle.train_step import OracleTrainer

N_RAYS = 64


@pytest.fixture(scope="module")
def grads():
    sconf, cconf, rconf = U.confs_from_kw(bench.SDF_KW, bench.COL_KW, bench.REN_KW)
    sp, cp, clip_sd, text = bench.synth_weights()
    hv = bench.WL.make_view(0, n_rays=N_RAYS, H=bench.CANVAS, W=bench.CANVAS, seed=0, bg_choice=3)
    orc = {dt: OracleTrainer(sconf, cconf, rconf, sp, cp, bench.VARIANCE, clip_sd, text, dtype=dt)
           for dt in (torch.float64, torch.float32)}
    with torch.no_grad():
        d = lambda t: t.double().reshape(t.shape[0], -1)
        z = neus.hierarchical_z(lambda x: neus.sdf_value(orc[torch.float64].sp, sconf, x), rconf, d(hv.rays_o),
                                d(hv.rays_d), d(hv.near), d(hv.far), d(hv.jitter)).float()
    r64 = S.oracle_step(orc[torch.float64], hv, z)
    r32 = S.oracle_step(orc[torch.float32], hv, z, d_canvases=r64["d_canvases"])
    return sconf, cconf, r32["injected"], r64["injected"]


def _scaled(g, keys, f, rows=slice(None), cols=slice(None)):
    g = {k: v.clone() for k, v in g.items()}
    for k in keys:
        if g[k].dim() == 0:
            g[k] *= f
        elif g[k].dim() == 2:
            g[k][rows, cols] *= f
        else:
            g[k][rows] *= f
    return g


LAST = f"sdf.lin{bench.SDF_KW['n_layers']}"
# name: (defect, slice that must be named, whether the flat rel-L2 of the gradient stays below 1e-3 at N_RAYS)
DEFECTS = {
    "extra_lin zeroed": (lambda g: _scaled(g, [k for k in g if k.startswith("col.extra_lin.")], 0.0),
                         "col.extra_lin.weight_v", True),
    "colour x 1.05": (lambda g: _scaled(g, [k for k in g if k.startswith("col.")], 1.05), "col.lin4.bias", True),
    "variance x 1.01": (lambda g: _scaled(g, ["var.variance"], 1.01), "var.variance", True),
    "sdf row x (1 + 1e-3)": (lambda g: _scaled(g, [f"{LAST}.{w}" for w in ("weight_v", "weight_g", "bias")], 1.0 + 1e-3,
                                               rows=slice(0, 1)), f"{LAST}.bias[sdf row]", True),
    "colour lin0 normal columns zeroed": (lambda g: _scaled(g, ["col.lin0.weight_v"], 0.0, cols=slice(3, 6)),
                                          "col.lin0.weight_v[normal cols]", True),
}


def test_fp32_oracle_passes_the_slice_bars(grads):
    sconf, cconf, g32, g64 = grads
    err, share = S.slice_errors(g32, g64, sconf, cconf)
    bars = S.bars("exact", "bench")
    S.report("fp32 oracle vs fp64, (a) bars of the benchmark networks", err, share, bars=bars)
    bad = S.failures(err, bars)
    assert not bad, bad


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_planted_defect_fails_on_its_slice(grads, defect):
    sconf, cconf, g32, g64 = grads
    plant, slice_name, flat_misses = DEFECTS[defect]
    bad_g = plant(g32)
    err, _ = S.slice_errors(bad_g, g64, sconf, cconf)
    bad = S.failures(err, S.bars("exact", "bench"))
    flat = U.flat_rel_l2(bad_g, g64)
    print(f"{defect}: flat rel-L2 {flat:.2e}; failing slices {bad}")
    assert any(b.startswith(slice_name + ":") for b in bad), bad
    assert (flat < 1e-3) == flat_misses
