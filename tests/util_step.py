"""Per-slice comparison of the appearance step's parameter gradient with the fp64 oracle step
(tests/test_step_at_scale_gpu.py, and its CPU self-check tests/test_step_slices_cpu.py).

A flat rel-L2 over the whole gradient is dominated by the SDF's weight_v and biases: the colour network holds about 1 % of
the benchmark gradient's norm and the extra-colour head about 1e-6 of it.  So the gradient is cut into slices -- every
parameter tensor, plus the rows and columns where distinct paths of the backward land -- and each slice is compared with
its own norm."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from oracle.train_step import OracleTrainer

import bench
import util_neus as U


def bench_confs():
    return U.confs_from_kw(bench.SDF_KW, bench.COL_KW, bench.REN_KW)


def slices(grads: Dict[str, torch.Tensor], sconf, cconf) -> Dict[str, torch.Tensor]:
    """name -> gradient slice (fp64, flat).  Every parameter tensor whole, and also:
    - the last SDF linear's row 0 (the sdf head: the eikonal and second-order paths land there) apart from its feature rows;
    - each skip linear's weight_v columns that read the hidden activations apart from those that read the encoding;
    - colour lin0's weight_v columns that read the point, the normal (the gradient-chain path) and the feature."""
    if cconf.mode != "no_view_dir":
        raise ValueError("slices: colour lin0 is cut as [points, normals, features] (mode no_view_dir)")
    g = {k: v.detach().double().cpu() for k, v in grads.items()}
    out = {k: v.reshape(-1) for k, v in g.items()}
    last = sconf.n_lin - 1
    for w in ("weight_v", "weight_g", "bias"):
        t = g[f"sdf.lin{last}.{w}"]
        out[f"sdf.lin{last}.{w}[sdf row]"] = t[:1].reshape(-1)
        out[f"sdf.lin{last}.{w}[feature rows]"] = t[1:].reshape(-1)
    for k in sconf.skip_in:
        if k < sconf.n_lin:
            t = g[f"sdf.lin{k}.weight_v"]
            h = t.shape[1] - sconf.d_enc                    # the skip concat is [hidden, encoding] / sqrt(2)
            out[f"sdf.lin{k}.weight_v[hidden cols]"] = t[:, :h].reshape(-1)
            out[f"sdf.lin{k}.weight_v[enc cols]"] = t[:, h:].reshape(-1)
    t = g["col.lin0.weight_v"]
    for name, cols in (("point", slice(0, 3)), ("normal", slice(3, 6)), ("feature", slice(6, None))):
        out[f"col.lin0.weight_v[{name} cols]"] = t[:, cols].reshape(-1)
    return out


def slice_errors(got: Dict[str, torch.Tensor], ref: Dict[str, torch.Tensor], sconf, cconf):
    """-> ({slice: rel-L2 of got against ref}, {slice: norm of ref's slice / norm of ref's flat gradient})."""
    gs, rs = slices(got, sconf, cconf), slices(ref, sconf, cconf)
    flat = math.sqrt(sum(rs[k].pow(2).sum().item() for k in ref))
    err = {k: (gs[k] - rs[k]).norm().item() / max(rs[k].norm().item(), 1e-300) for k in rs}
    share = {k: rs[k].norm().item() / flat for k in rs}
    return err, share


def failures(err: Dict[str, float], bars: Dict[str, float], floor: Optional[Dict[str, float]] = None) -> List[str]:
    """The slices whose error exceeds max(bar, 10 x the fp32 oracle's error on the slice), as readable strings."""
    bad = []
    for k, e in err.items():
        bar = bars.get(k, 0.0)
        if floor is not None:
            bar = max(bar, 10.0 * floor[k])
        if not e <= bar:
            bad.append(f"{k}: {e:.3e} > bar {bar:.1e}")
    return bad


def report(title: str, err, share, floor=None, bars=None):
    """One printed line per slice: error, fp32-oracle floor, share of the flat norm, bar."""
    print(f"---- {title}")
    for k in err:
        f = "" if floor is None else f"  fp32 floor {floor[k]:.2e}"
        b = "" if bars is None else f"  bar {bars.get(k, 0.0):.0e}"
        print(f"  {k:38s} err {err[k]:.3e}{f}  share {share[k]:.2e}{b}")


def oracle_step(orc: OracleTrainer, view, z_vals: torch.Tensor, d_canvases: Optional[torch.Tensor] = None):
    """The oracle step on the given depths.  Returns a dict with
    - ``loss``, ``cos``: the step's loss and its two CLIP cosines;
    - ``d_canvases``: the gradient of the CLIP terms at the oracle's own canvases [2,H,W,3], rounded to fp32;
    - ``step``: {param name: gradient of the whole loss};
    - ``injected``: {param name: gradient of base loss + sum(d_canvases . canvases)}, where d_canvases is the argument, or
      this run's own ``d_canvases`` when it is None -- the step with the CLIP tower's cotangent held fixed."""
    total, aux = orc.loss(view, z_vals=z_vals)
    st = aux["stage"]
    canv = [st["texture_canvas"], st["shading_canvas"]]
    params = [v for _, v in orc.named_params()]
    names = [k for k, _ in orc.named_params()]

    def named(gs):
        return {k: (torch.zeros_like(v) if g is None else g).detach() for k, v, g in zip(names, params, gs)}

    dc = torch.stack(torch.autograd.grad(total - st["base_loss"], canv, retain_graph=True)).float()
    d = dc if d_canvases is None else d_canvases
    obj = st["base_loss"] + sum((d[i].to(orc.dtype) * canv[i]).sum() for i in range(2))
    injected = named(torch.autograd.grad(obj, params, retain_graph=True, allow_unused=True))
    step = named(torch.autograd.grad(total, params, allow_unused=True))
    return {"loss": total.item(), "cos": aux["cos"].detach().double(), "d_canvases": dc, "step": step,
            "injected": injected}


# Per-slice bars measured on an H100 (see the docstring of tests/test_step_at_scale_gpu.py and DESIGN §5), by comparison
# ("exact" = (a), "step" = (b), "replay" = replayed against eager gradient) and network size ("bench", "shipped").
BARS = {
    "exact": {
        "bench": {
            "sdf.lin0.bias": 2e-04, "sdf.lin0.weight_g": 2e-04, "sdf.lin0.weight_v": 2e-04, "sdf.lin1.bias": 2e-04,
            "sdf.lin1.weight_g": 2e-04, "sdf.lin1.weight_v": 2e-04, "sdf.lin2.bias": 2e-04, "sdf.lin2.weight_g": 2e-04,
            "sdf.lin2.weight_v": 2e-04, "sdf.lin3.bias": 2e-04, "sdf.lin3.weight_g": 2e-04, "sdf.lin3.weight_v": 2e-04,
            "sdf.lin4.bias": 1e-04, "sdf.lin4.weight_g": 2e-04, "sdf.lin4.weight_v": 1e-04, "sdf.lin5.bias": 1e-04,
            "sdf.lin5.weight_g": 2e-04, "sdf.lin5.weight_v": 1e-04, "sdf.lin6.bias": 1e-04, "sdf.lin6.weight_g": 1e-04,
            "sdf.lin6.weight_v": 1e-04, "sdf.lin7.bias": 1e-04, "sdf.lin7.weight_g": 1e-04, "sdf.lin7.weight_v": 1e-04,
            "sdf.lin8.bias": 1e-04, "sdf.lin8.weight_g": 1e-04, "sdf.lin8.weight_v": 1e-04, "col.lin0.bias": 5e-04,
            "col.lin0.weight_g": 5e-04, "col.lin0.weight_v": 5e-04, "col.lin1.bias": 5e-04, "col.lin1.weight_g": 5e-04,
            "col.lin1.weight_v": 5e-04, "col.lin2.bias": 2e-04, "col.lin2.weight_g": 1e-04, "col.lin2.weight_v": 2e-04,
            "col.lin3.bias": 5e-05, "col.lin3.weight_g": 5e-05, "col.lin3.weight_v": 5e-05, "col.lin4.bias": 5e-05,
            "col.lin4.weight_g": 5e-05, "col.lin4.weight_v": 5e-05, "col.extra_lin.bias": 5e-05,
            "col.extra_lin.weight_g": 1e-04, "col.extra_lin.weight_v": 5e-05, "var.variance": 1e-04,
            "sdf.lin8.weight_v[sdf row]": 1e-04, "sdf.lin8.weight_v[feature rows]": 5e-04,
            "sdf.lin8.weight_g[sdf row]": 1e-04, "sdf.lin8.weight_g[feature rows]": 5e-04,
            "sdf.lin8.bias[sdf row]": 1e-04, "sdf.lin8.bias[feature rows]": 5e-04,
            "sdf.lin4.weight_v[hidden cols]": 2e-04, "sdf.lin4.weight_v[enc cols]": 1e-04,
            "col.lin0.weight_v[point cols]": 5e-04, "col.lin0.weight_v[normal cols]": 5e-04,
            "col.lin0.weight_v[feature cols]": 5e-04,
        },
        "shipped": {
            "sdf.lin0.bias": 1e-03, "sdf.lin0.weight_g": 1e-03, "sdf.lin0.weight_v": 1e-03, "sdf.lin1.bias": 1e-03,
            "sdf.lin1.weight_g": 1e-03, "sdf.lin1.weight_v": 1e-03, "sdf.lin2.bias": 1e-03, "sdf.lin2.weight_g": 1e-03,
            "sdf.lin2.weight_v": 1e-03, "sdf.lin3.bias": 5e-04, "sdf.lin3.weight_g": 5e-04, "sdf.lin3.weight_v": 1e-03,
            "sdf.lin4.bias": 5e-04, "sdf.lin4.weight_g": 2e-04, "sdf.lin4.weight_v": 1e-03, "col.lin0.bias": 5e-04,
            "col.lin0.weight_g": 5e-04, "col.lin0.weight_v": 5e-04, "col.lin1.bias": 2e-04, "col.lin1.weight_g": 5e-04,
            "col.lin1.weight_v": 5e-04, "col.lin2.bias": 5e-06, "col.lin2.weight_g": 1e-04, "col.lin2.weight_v": 2e-05,
            "col.extra_lin.bias": 1e-05, "col.extra_lin.weight_g": 2e-05, "col.extra_lin.weight_v": 5e-05,
            "var.variance": 1e-03, "sdf.lin4.weight_v[sdf row]": 1e-03, "sdf.lin4.weight_v[feature rows]": 5e-04,
            "sdf.lin4.weight_g[sdf row]": 2e-04, "sdf.lin4.weight_g[feature rows]": 5e-04,
            "sdf.lin4.bias[sdf row]": 5e-04, "sdf.lin4.bias[feature rows]": 5e-04,
            "sdf.lin4.weight_v[hidden cols]": 1e-03, "sdf.lin4.weight_v[enc cols]": 1e-03,
            "col.lin0.weight_v[point cols]": 5e-04, "col.lin0.weight_v[normal cols]": 5e-04,
            "col.lin0.weight_v[feature cols]": 1e-03,
        },
    },
    "step": {
        "bench": {
            "sdf.lin0.bias": 2e-04, "sdf.lin0.weight_g": 2e-04, "sdf.lin0.weight_v": 2e-04, "sdf.lin1.bias": 2e-04,
            "sdf.lin1.weight_g": 2e-04, "sdf.lin1.weight_v": 2e-04, "sdf.lin2.bias": 2e-04, "sdf.lin2.weight_g": 2e-04,
            "sdf.lin2.weight_v": 2e-04, "sdf.lin3.bias": 2e-04, "sdf.lin3.weight_g": 2e-04, "sdf.lin3.weight_v": 2e-04,
            "sdf.lin4.bias": 1e-04, "sdf.lin4.weight_g": 2e-04, "sdf.lin4.weight_v": 1e-04, "sdf.lin5.bias": 1e-04,
            "sdf.lin5.weight_g": 2e-04, "sdf.lin5.weight_v": 2e-04, "sdf.lin6.bias": 1e-04, "sdf.lin6.weight_g": 1e-04,
            "sdf.lin6.weight_v": 1e-04, "sdf.lin7.bias": 1e-04, "sdf.lin7.weight_g": 2e-04, "sdf.lin7.weight_v": 1e-04,
            "sdf.lin8.bias": 1e-04, "sdf.lin8.weight_g": 1e-04, "sdf.lin8.weight_v": 1e-04, "col.lin0.bias": 5e-04,
            "col.lin0.weight_g": 5e-04, "col.lin0.weight_v": 5e-04, "col.lin1.bias": 5e-04, "col.lin1.weight_g": 5e-04,
            "col.lin1.weight_v": 5e-04, "col.lin2.bias": 2e-04, "col.lin2.weight_g": 1e-04, "col.lin2.weight_v": 2e-04,
            "col.lin3.bias": 5e-05, "col.lin3.weight_g": 5e-05, "col.lin3.weight_v": 5e-05, "col.lin4.bias": 5e-05,
            "col.lin4.weight_g": 5e-05, "col.lin4.weight_v": 5e-05, "col.extra_lin.bias": 1e-02,
            "col.extra_lin.weight_g": 1e-02, "col.extra_lin.weight_v": 1e-02, "var.variance": 1e-04,
            "sdf.lin8.weight_v[sdf row]": 1e-04, "sdf.lin8.weight_v[feature rows]": 5e-04,
            "sdf.lin8.weight_g[sdf row]": 1e-04, "sdf.lin8.weight_g[feature rows]": 5e-04,
            "sdf.lin8.bias[sdf row]": 1e-04, "sdf.lin8.bias[feature rows]": 5e-04,
            "sdf.lin4.weight_v[hidden cols]": 2e-04, "sdf.lin4.weight_v[enc cols]": 1e-04,
            "col.lin0.weight_v[point cols]": 5e-04, "col.lin0.weight_v[normal cols]": 5e-04,
            "col.lin0.weight_v[feature cols]": 5e-04,
        },
        "shipped": {
            "sdf.lin0.bias": 1e-03, "sdf.lin0.weight_g": 2e-03, "sdf.lin0.weight_v": 1e-03, "sdf.lin1.bias": 1e-03,
            "sdf.lin1.weight_g": 2e-03, "sdf.lin1.weight_v": 2e-03, "sdf.lin2.bias": 1e-03, "sdf.lin2.weight_g": 1e-03,
            "sdf.lin2.weight_v": 1e-03, "sdf.lin3.bias": 1e-03, "sdf.lin3.weight_g": 1e-03, "sdf.lin3.weight_v": 1e-03,
            "sdf.lin4.bias": 5e-04, "sdf.lin4.weight_g": 2e-04, "sdf.lin4.weight_v": 1e-03, "col.lin0.bias": 5e-04,
            "col.lin0.weight_g": 5e-04, "col.lin0.weight_v": 5e-04, "col.lin1.bias": 5e-04, "col.lin1.weight_g": 5e-04,
            "col.lin1.weight_v": 5e-04, "col.lin2.bias": 5e-06, "col.lin2.weight_g": 1e-04, "col.lin2.weight_v": 2e-05,
            "col.extra_lin.bias": 1e-02, "col.extra_lin.weight_g": 1e-02, "col.extra_lin.weight_v": 1e-02,
            "var.variance": 1e-03, "sdf.lin4.weight_v[sdf row]": 1e-03, "sdf.lin4.weight_v[feature rows]": 5e-04,
            "sdf.lin4.weight_g[sdf row]": 2e-04, "sdf.lin4.weight_g[feature rows]": 5e-04,
            "sdf.lin4.bias[sdf row]": 5e-04, "sdf.lin4.bias[feature rows]": 5e-04,
            "sdf.lin4.weight_v[hidden cols]": 1e-03, "sdf.lin4.weight_v[enc cols]": 1e-03,
            "col.lin0.weight_v[point cols]": 5e-04, "col.lin0.weight_v[normal cols]": 5e-04,
            "col.lin0.weight_v[feature cols]": 1e-03,
        },
    },
    "replay": {
        "bench": {
            "sdf.lin0.weight_g": 1e-04, "sdf.lin0.weight_v": 5e-05, "sdf.lin0.bias": 5e-05, "sdf.lin1.weight_g": 5e-05,
            "sdf.lin1.weight_v": 5e-05, "sdf.lin1.bias": 5e-05, "sdf.lin2.weight_g": 5e-05, "sdf.lin2.weight_v": 5e-05,
            "sdf.lin2.bias": 5e-05, "sdf.lin3.weight_g": 5e-05, "sdf.lin3.weight_v": 5e-05, "sdf.lin3.bias": 5e-05,
            "sdf.lin4.weight_g": 5e-05, "sdf.lin4.weight_v": 5e-05, "sdf.lin4.bias": 5e-05, "sdf.lin5.weight_g": 5e-05,
            "sdf.lin5.weight_v": 5e-05, "sdf.lin5.bias": 5e-05, "sdf.lin6.weight_g": 5e-05, "sdf.lin6.weight_v": 5e-05,
            "sdf.lin6.bias": 2e-05, "sdf.lin7.weight_g": 2e-05, "sdf.lin7.weight_v": 5e-05, "sdf.lin7.bias": 2e-05,
            "sdf.lin8.weight_g": 5e-06, "sdf.lin8.weight_v": 2e-05, "sdf.lin8.bias": 5e-06, "col.lin0.weight_g": 1e-05,
            "col.lin0.weight_v": 1e-05, "col.lin0.bias": 1e-05, "col.lin1.weight_g": 1e-05, "col.lin1.weight_v": 1e-05,
            "col.lin1.bias": 1e-05, "col.lin2.weight_g": 1e-05, "col.lin2.weight_v": 1e-05, "col.lin2.bias": 1e-05,
            "col.lin3.weight_g": 1e-05, "col.lin3.weight_v": 1e-05, "col.lin3.bias": 1e-05, "col.lin4.weight_g": 2e-06,
            "col.lin4.weight_v": 2e-06, "col.lin4.bias": 2e-06, "col.extra_lin.weight_g": 2e-02,
            "col.extra_lin.weight_v": 1e-02, "col.extra_lin.bias": 1e-02, "var.variance": 5e-06,
            "sdf.lin8.weight_v[sdf row]": 2e-05, "sdf.lin8.weight_v[feature rows]": 2e-05,
            "sdf.lin8.weight_g[sdf row]": 5e-06, "sdf.lin8.weight_g[feature rows]": 2e-05,
            "sdf.lin8.bias[sdf row]": 5e-06, "sdf.lin8.bias[feature rows]": 2e-05,
            "sdf.lin4.weight_v[hidden cols]": 5e-05, "sdf.lin4.weight_v[enc cols]": 5e-05,
            "col.lin0.weight_v[point cols]": 2e-05, "col.lin0.weight_v[normal cols]": 2e-05,
            "col.lin0.weight_v[feature cols]": 1e-05,
        },
        "shipped": {
            "sdf.lin0.weight_g": 1e-03, "sdf.lin0.weight_v": 1e-03, "sdf.lin0.bias": 1e-03, "sdf.lin1.weight_g": 1e-03,
            "sdf.lin1.weight_v": 1e-03, "sdf.lin1.bias": 1e-03, "sdf.lin2.weight_g": 1e-03, "sdf.lin2.weight_v": 1e-03,
            "sdf.lin2.bias": 5e-04, "sdf.lin3.weight_g": 1e-03, "sdf.lin3.weight_v": 1e-03, "sdf.lin3.bias": 5e-04,
            "sdf.lin4.weight_g": 1e-04, "sdf.lin4.weight_v": 1e-03, "sdf.lin4.bias": 2e-05, "col.lin0.weight_g": 5e-04,
            "col.lin0.weight_v": 5e-04, "col.lin0.bias": 5e-04, "col.lin1.weight_g": 2e-04, "col.lin1.weight_v": 2e-04,
            "col.lin1.bias": 2e-04, "col.lin2.weight_g": 1e-05, "col.lin2.weight_v": 2e-06, "col.lin2.bias": 1e-06,
            "col.extra_lin.weight_g": 2e-02, "col.extra_lin.weight_v": 1e-02, "col.extra_lin.bias": 1e-02,
            "var.variance": 5e-05, "sdf.lin4.weight_v[sdf row]": 1e-03, "sdf.lin4.weight_v[feature rows]": 5e-04,
            "sdf.lin4.weight_g[sdf row]": 1e-04, "sdf.lin4.weight_g[feature rows]": 5e-04,
            "sdf.lin4.bias[sdf row]": 2e-05, "sdf.lin4.bias[feature rows]": 5e-04,
            "sdf.lin4.weight_v[hidden cols]": 1e-03, "sdf.lin4.weight_v[enc cols]": 1e-03,
            "col.lin0.weight_v[point cols]": 5e-04, "col.lin0.weight_v[normal cols]": 5e-04,
            "col.lin0.weight_v[feature cols]": 2e-04,
        },
    },
}


def bars(kind: str, config: str) -> Dict[str, float]:
    return BARS.get(kind, {}).get("bench" if config.startswith("bench") else "shipped", {})
