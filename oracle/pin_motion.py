"""Pin oracle/motion.py against the reference's own motion stage (AvatarAnimate/models/motion_generation.py, builder.py,
main.py) run in THIS container on the CPU, and record what it computed as tests/golden/ref_motion_small.pt.

main.py and the generators import ``clip``, ``smplx``, ``human_body_prior``, ``neural_renderer``, ``pyhocon``, ``tqdm``
and ``visualize``, none of which is installed.  This script puts stand-ins for them in ``sys.modules`` and imports the
UNMODIFIED files:
  * ``clip``: ``load`` returns a model whose ``encode_text`` is a fixed seeded feature (the motion stage's CLIP term is
    off, and VPoserCodebook only needs a feature its codebook is built around);
  * ``smplx.create``: a placeholder module (nothing on these paths poses SMPL);
  * ``human_body_prior``: ``load_model`` returns a VPoser whose ``decode`` is oracle/animate.py's and whose ``encode``
    is oracle/motion.py's (``.mean``), on seeded weights (PARITY UNPINNED, the package is absent);
  * ``neural_renderer``: ``load_obj`` for render.py's import-time texture load (never rendered with);
  * ``pyhocon``: avatarclip_b200/conf.py's reader; ``tqdm``; ``visualize``: main.py's jpg / mp4 writers, no-ops.
torch's ``"cuda"`` device is mapped to the CPU.  The motion VAE checkpoint holds oracle/motion.py's full-size seeded
decoder (latent 256, 4 layers, 4 heads, FF 1024, 330 outputs) and no encoder keys; the reference loads it with
``strict=False``.  Three confs run through ``main.main``: MotionInterpolation with its defaults, and MotionOptimizer
with clip_coef = 0 for NUM_ITER iterations, once with delta_coef = 0 and recon_coef all 1 (the baseline confs) and once
with delta_coef = 0.01 and the default recon_coef.  Recorded: the seeds, the candidate poses, the interpolated motion,
and per optimiser run the initial latent (``torch.randn`` inside get_motion), every iteration's loss, the final latent
and motion; and the loss of oracle/motion.py's fp32 loop over 5000 iterations from the baseline run's initial latent.
Nothing of the reference is copied into this repository.

    python -m oracle.pin_motion
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

REF = "/root/reference/AvatarAnimate"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TORCH_SEED = 7
TEXT_SEED = 8
NUM_ITER = 50
LONG_ITER = 5000
RUNS = {"interpolation": "type = MotionInterpolation",
        "delta0": "type = MotionOptimizer\n    num_iteration = %d\n    clip_coef = 0.0\n    delta_coef = 0.0\n"
                  "    recon_coef = [1.0, 1.0, 1.0, 1.0, 1.0]" % NUM_ITER,
        "delta": "type = MotionOptimizer\n    num_iteration = %d\n    clip_coef = 0.0\n    delta_coef = 0.01" % NUM_ITER}


def text_feature() -> torch.Tensor:
    return torch.randn(512, generator=torch.Generator().manual_seed(TEXT_SEED))


def main():
    from oracle import animate as OA
    from oracle import motion as OM
    import torch._dynamo  # noqa: F401  (imported before the stand-ins: it looks up installed modules' specs)
    sys.path.insert(0, ROOT)
    vp_sd, enc_sd, vae_sd = OA.vposer_state(), OM.vposer_encoder_state(), OM.motion_vae_state()
    tf = text_feature()
    rec = {"adam": [], "losses": []}

    _tto, _mto = torch.Tensor.to, torch.nn.Module.to
    cpu = lambda a: tuple("cpu" if (isinstance(x, str) and x.startswith("cuda")) else x for x in a)
    torch.Tensor.to = lambda self, *a, **k: _tto(self, *cpu(a), **{kk: ("cpu" if kk == "device" else v)
                                                                   for kk, v in k.items()})
    torch.nn.Module.to = lambda self, *a, **k: _mto(self, *cpu(a), **{kk: ("cpu" if kk == "device" else v)
                                                                      for kk, v in k.items()})
    torch.cuda.is_available = lambda: True
    torch.cuda.is_current_stream_capturing = lambda: False     # Adam.step's check, reached through is_available

    class Perceptor:
        def eval(self):
            return self

        def encode_text(self, tokens):
            return tf[None].clone()

    clip = types.ModuleType("clip")
    clip.load = lambda name, device=None, jit=False: (Perceptor(), None)
    clip.tokenize = lambda s: torch.zeros(1, 77, dtype=torch.long)
    smplx = types.ModuleType("smplx")
    smplx.create = lambda path, model_type: torch.nn.Module()

    class VPoser(torch.nn.Module):
        def decode(self, z):
            pose, rot = OA.vposer_decode(z, vp_sd)
            return {"pose_body": torch.from_numpy(pose).float(),
                    "pose_body_matrot": torch.from_numpy(rot.reshape(z.shape[0], -1, 9)).float()}

        def encode(self, x):
            return types.SimpleNamespace(mean=OM.vposer_encode(x, enc_sd).float())

    hbp = types.ModuleType("human_body_prior")
    tools = types.ModuleType("human_body_prior.tools")
    loader = types.ModuleType("human_body_prior.tools.model_loader")
    loader.load_model = lambda path, model_code=None, remove_words_in_model_weights=None, disable_grad=False: (
        VPoser(), None)
    models = types.ModuleType("human_body_prior.models")
    vpm = types.ModuleType("human_body_prior.models.vposer_model")
    vpm.VPoser = VPoser
    nr = types.ModuleType("neural_renderer")
    nr.load_obj = lambda fname, load_texture=True, texture_size=8: (None, None, None)
    tqdm = types.ModuleType("tqdm")
    tqdm.tqdm = lambda it, *a, **k: it
    visualize = types.ModuleType("visualize")
    visualize.render_pose = lambda pose, path: None
    visualize.render_motion = lambda motion, path: None
    from avatarclip_b200 import conf as conf_mod
    pyhocon = types.ModuleType("pyhocon")
    pyhocon.ConfigFactory = types.SimpleNamespace(parse_string=conf_mod.parse_string)
    sys.modules.update({"pyhocon": pyhocon, "clip": clip, "smplx": smplx, "human_body_prior": hbp,
                        "human_body_prior.tools": tools, "human_body_prior.tools.model_loader": loader,
                        "human_body_prior.models": models, "human_body_prior.models.vposer_model": vpm,
                        "neural_renderer": nr, "tqdm": tqdm, "visualize": visualize})

    class RecordingAdam(torch.optim.Adam):
        def __init__(self, params, **kw):
            params = list(params)
            rec["adam"].append(dict(init=params[0].detach().clone(), param=params[0], cfg=kw))
            super().__init__(params, **kw)

    _backward = torch.Tensor.backward

    def backward(self, *a, **k):
        if self.dim() == 0:
            rec["losses"].append(float(self.detach()))
        return _backward(self, *a, **k)

    torch.optim.Adam = RecordingAdam
    torch.Tensor.backward = backward

    cwd = os.getcwd()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data"))
        torch.save(OA.make_codebook(tf), os.path.join(tmp, "data", "codebook.pth"))
        torch.save({"state_dict": vae_sd}, os.path.join(tmp, "data", "motion_vae.pth"))
        os.chdir(tmp)
        sys.path.insert(0, REF)
        try:
            import main as ref_main
            for name, block in RUNS.items():
                rec["adam"], rec["losses"] = [], []
                p = os.path.join(tmp, f"{name}.conf")
                with open(p, "w") as fp:
                    fp.write(f"general {{\n    base_exp_dir = {tmp}/exp_{name}\n    mode = motion\n    text = {OA.TEXT}\n"
                             f"}}\n\npose_generator {{\n    type = VPoserCodebook\n}}\n\nmotion_generator {{\n    {block}\n}}\n")
                torch.manual_seed(TORCH_SEED)
                ref_main.main(p)
                d = f"{tmp}/exp_{name}"
                r = dict(poses=torch.stack([torch.from_numpy(np.load(f"{d}/candidate_{i}.npy")) for i in range(5)]),
                         motion=torch.from_numpy(np.load(f"{d}/motion.npy")))
                if rec["adam"]:
                    a = rec["adam"][0]
                    r.update(latent_init=a["init"], latent=a["param"].detach().clone(), optim_cfg=a["cfg"],
                             loss=torch.tensor(rec["losses"]))
                out[name] = r
        finally:
            os.chdir(cwd)
            torch.Tensor.backward = _backward

    # ---- the restatement against the reference
    poses = out["interpolation"]["poses"]
    m = OM.interpolation_motion(poses, enc_sd, vp_sd)
    e = np.abs(m - out["interpolation"]["motion"][:, :63].double().numpy()).max()
    print(f"[pin_motion] interpolation: motion {tuple(out['interpolation']['motion'].shape)}, oracle err {e:.2e}")
    assert e <= 1e-4 and out["interpolation"]["motion"][:, 63:].abs().max() == 0
    cfgs = {"delta0": ([1.0] * 5, 0.0), "delta": ([1, 0.8, 0.6, 0.4, 0.2], 0.01)}
    for name, (coef, dc) in cfgs.items():
        r = out[name]
        assert torch.equal(r["poses"], poses) and len(r["loss"]) == NUM_ITER
        l64, z64, m64 = OM.optimize(vae_sd, r["poses"], r["latent_init"], NUM_ITER, coef, dc)
        l32, _, _ = OM.optimize(vae_sd, r["poses"], r["latent_init"], NUM_ITER, coef, dc, dtype=torch.float32)
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
        print(f"[pin_motion] {name}: loss {r['loss'][0]:.5f} -> {r['loss'][-1]:.5f}; oracle fp64 vs reference: loss "
              f"{rel(r['loss'].double(), l64):.2e}, latent {rel(r['latent'].double(), z64):.2e}, motion "
              f"{rel(r['motion'][:, :63].double(), m64):.2e}; oracle fp32 vs fp64 loss {rel(l32, l64):.2e}")
        assert rel(r["loss"].double(), l64) <= 1e-3 and r["loss"][-1] < r["loss"][0]

    # the long run the device is held to: the oracle's fp32 CPU loop over the shipped 5000 iterations (baseline conf)
    r, (coef, dc) = out["delta0"], cfgs["delta0"]
    l_long, _, _ = OM.optimize(vae_sd, r["poses"], r["latent_init"], LONG_ITER, coef, dc, dtype=torch.float32)
    print(f"[pin_motion] oracle fp32, {LONG_ITER} iterations: final loss {l_long[-1]:.6f}")

    rec_out = dict(text=OA.TEXT, long_iter=LONG_ITER, oracle_fp32_long_loss=l_long.float(), torch_seed=TORCH_SEED, num_iter=NUM_ITER,
                   seeds=dict(vposer=OA.VPOSER_SEED, encoder=OM.ENCODER_SEED, motion_vae=OM.MOTION_VAE_SEED,
                              codebook=OA.CODEBOOK_SEED, text=TEXT_SEED),
                   poses=poses, interpolation=out["interpolation"]["motion"],
                   optimizer={n: {k: out[n][k] for k in ("latent_init", "loss", "latent", "motion")} for n in cfgs},
                   optimizer_conf={n: dict(recon_coef=c, delta_coef=d, lr=0.01) for n, (c, d) in cfgs.items()})
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(rec_out, os.path.join(GOLDEN, "ref_motion_small.pt"))


if __name__ == "__main__":
    main()
