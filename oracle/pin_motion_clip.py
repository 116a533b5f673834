"""Pin AvatarAnimate's MotionOptimizer with its CLIP term against the reference's own code
(AvatarAnimate/models/motion_generation.py, builder.py, main.py) run in THIS container on the CPU, and record what it
computed as tests/golden/ref_motion_clip_small.pt.

As oracle/pin_motion.py and oracle/pin_pose_optimizer.py do, this script puts stand-ins for the packages the reference
imports in ``sys.modules`` and imports the UNMODIFIED files.  The stand-ins are the ones those two scripts use:
  * ``human_body_prior``: a VPoser whose ``decode`` is oracle/animate.py's, on seeded weights (VPoserCodebook's
    candidates; its codebook is oracle/animate.py's make_codebook around the text feature);
  * ``smplx.create``: SMPL with zero betas through torch fp64 autograd of oracle/lbs.py's my_lbs (the shipped template,
    synthetic SMPL tensors of oracle/drive.py golden_smpl);
  * ``neural_renderer.Renderer``: an autograd Function whose forward is oracle/shapegen.py's textured render and whose
    backward is oracle/pose_optimizer.py's restatement of neural_renderer's backward on that render's maps;
  * ``clip``: the oracle CLIP towers (oracle/clip_text.py, oracle/clip_vit.py) on seeded weights;
  * ``pyhocon``, ``tqdm``, ``visualize``.
The motion VAE checkpoint holds oracle/motion.py's full-size seeded decoder.  torch's ``"cuda"`` device is mapped to
the CPU.  ``torch.optim.Adam`` records each step's parameter and gradient, ``np.random.randint`` each draw, the
renderer each camera and ``Tensor.backward`` each loss.

Two runs of main.main on a MotionOptimizer conf with NUM_ITER iterations each:
  * ``shipped``: the reference's coefficients (recon_coef (1, 0.8, 0.6, 0.4, 0.2), clip_coef 0.001, delta_coef 0.01,
    clip_num_part 30);
  * ``clip_only``: recon_coef all 0, delta_coef 0 and clip_coef 1, so that the latent gradient is the CLIP term alone.
What this pins: the draws and their order (torch.randn for the latent, then per iteration np.random.randint and the
camera's np.random.randn), the scored frames and their weights, the loss, Adam and the written files.  What it does not
pin: the rasteriser's gradient itself, which is this project's restatement (neural_renderer is absent).  Nothing of the
reference is copied into this repository.

    python -m oracle.pin_motion_clip
"""
import importlib
import os
import sys
import tempfile
import types

import numpy as np
import torch

REF = "/root/reference/AvatarAnimate"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NP_SEED = 25
TORCH_SEED = 26
NUM_ITER = 4
RUNS = {"shipped": dict(num_iteration=NUM_ITER),
        "clip_only": dict(num_iteration=NUM_ITER, recon_coef=[0.0] * 5, delta_coef=0.0, clip_coef=1.0)}


def main():
    from oracle import animate as O
    from oracle import clip_text as oct
    from oracle import clip_vit as ocv
    from oracle import drive as D
    from oracle import lbs as olbs
    from oracle import motion as OM
    from oracle import pose_optimizer as OP
    from oracle import shapegen as OS
    sys.path.insert(0, ROOT)
    from avatarclip_b200.clip_tokenizer import ClipTokenizer

    tv, tf = D.template_obj()
    smpl = D.golden_smpl()
    visual, text = OS.clip_states()
    vis = {k[len("visual."):]: v for k, v in visual.items()}
    vp_sd, vae_sd = O.vposer_state(), OM.motion_vae_state()
    rec = {}

    # ---- stand-ins
    _tto, _mto = torch.Tensor.to, torch.nn.Module.to
    cpu = lambda a: tuple("cpu" if (isinstance(x, str) and x.startswith("cuda")) else x for x in a)
    torch.Tensor.to = lambda self, *a, **k: _tto(self, *cpu(a), **{kk: ("cpu" if kk == "device" else v)
                                                                   for kk, v in k.items()})
    torch.nn.Module.to = lambda self, *a, **k: _mto(self, *cpu(a), **{kk: ("cpu" if kk == "device" else v)
                                                                      for kk, v in k.items()})
    _avail = torch.cuda.is_available
    torch.cuda.is_available = lambda: True
    tok_holder = {}

    class Perceptor:
        def eval(self):
            return self

        def encode_text(self, tokens):
            return oct.encode_text(text, tokens.long())

        def encode_image(self, images):
            return ocv.encode_image(vis, images.float())

    clip = types.ModuleType("clip")
    clip.load = lambda name, device=None, jit=False: (Perceptor(), None)
    clip.tokenize = lambda s: tok_holder["tok"].tokenize(s[0] if isinstance(s, list) else s).long()

    dt = torch.float64
    sm = {k: torch.as_tensor(np.asarray(v)) for k, v in smpl.items()}

    class SMPLLayer(torch.nn.Module):
        faces = tf.astype(np.int64)

        def forward(self, body_pose, global_orient):
            bs = body_pose.shape[0]
            full = torch.cat([global_orient.to(dt), body_pose.to(dt)], 1)
            v, _ = olbs.my_lbs(sm["v_template"].to(dt)[None].expand(bs, -1, -1), full, sm["posedirs"].to(dt),
                               sm["J_regressor"].to(dt), sm["parents"].long(), sm["lbs_weights"].to(dt))
            return types.SimpleNamespace(vertices=v.float())

    smplx = types.ModuleType("smplx")
    smplx.create = lambda path, model_type: SMPLLayer()

    class VPoser(torch.nn.Module):
        def decode(self, z):
            pose, rot = O.vposer_decode(z, vp_sd)
            return {"pose_body": torch.from_numpy(pose).float(),
                    "pose_body_matrot": torch.from_numpy(rot.reshape(z.shape[0], -1, 9)).float()}

    hbp = types.ModuleType("human_body_prior")
    tools = types.ModuleType("human_body_prior.tools")
    loader = types.ModuleType("human_body_prior.tools.model_loader")
    loader.load_model = lambda path, model_code=None, remove_words_in_model_weights=None, disable_grad=False: (
        VPoser(), None)
    models = types.ModuleType("human_body_prior.models")
    vpm = types.ModuleType("human_body_prior.models.vposer_model")
    vpm.VPoser = VPoser

    class RasterFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, vertices, faces, textures, eye, n):
            v = vertices.detach().double().numpy()
            imgs, maps = [], []
            for b in range(v.shape[0]):
                rgb, fidx, rgb_ss, proj = OP.raster_maps(v[b], faces[b].numpy(), textures[b].double().numpy(), eye, n)
                maps.append((fidx, rgb_ss, proj))
                imgs.append(torch.from_numpy(rgb))
            ctx.save = (v, faces[0].numpy(), eye, maps)
            return torch.stack(imgs).permute(0, 3, 1, 2).float()

        @staticmethod
        def backward(ctx, g):
            v, faces, eye, maps = ctx.save
            e, rot = OS.look_at_camera(eye)
            rec["in_raster"] = True         # the light's backward is autograd: not a loss of the loop
            gv = np.stack([OP.raster_backward_image(v[b], faces, proj, e, rot, fidx, rgb_ss,
                                                    g[b].permute(1, 2, 0).double().numpy(), 2)
                           for b, (fidx, rgb_ss, proj) in enumerate(maps)])
            rec["in_raster"] = False
            return torch.from_numpy(gv).float(), None, None, None, None

    class Renderer:
        def __init__(self, camera_mode="look_at", image_size=256):
            assert camera_mode == "look_at"
            self.image_size, self.eye = image_size, None

        def to(self, device):
            return self

        def __call__(self, vertices, faces, textures):
            rec["rows"].append(vertices.shape[0])
            return RasterFn.apply(vertices, faces, textures, np.asarray(self.eye, dtype=np.float64),
                                  self.image_size), None, None

    def get_points_from_angles(d, el, az):
        rec["elevation"].append(float(el))
        rec["azimuth"].append(float(az))
        return O.eye(el, az)

    nr = types.ModuleType("neural_renderer")
    nr.load_obj = lambda fname, load_texture=True, texture_size=8: (
        None, None, torch.from_numpy(OS.load_obj_textures(fname, texture_size)).float())
    nr.Renderer = Renderer
    nr.get_points_from_angles = get_points_from_angles
    tqdm = types.ModuleType("tqdm")
    tqdm.tqdm = lambda it, *a, **k: it
    visualize = types.ModuleType("visualize")
    visualize.render_pose = lambda pose, path: None
    visualize.render_motion = lambda motion, path: None

    class RecordingAdam(torch.optim.Adam):
        def __init__(self, params, **kw):
            params = list(params)
            rec["init"], rec["param_obj"] = params[0].detach().clone(), params[0]
            rec["optim_cfg"] = dict(kw)
            super().__init__(params, **kw)

        def step(self, closure=None):
            p = self.param_groups[0]["params"][0]
            rec["param"].append(p.detach().clone())
            rec["grad"].append(p.grad.detach().clone())
            torch.cuda.is_available = _avail        # the step itself runs torch's CPU Adam
            try:
                return super().step(closure)
            finally:
                torch.cuda.is_available = lambda: True

    _randint = np.random.randint

    def randint(*a, **k):
        r = _randint(*a, **k)
        rec["st_idx"].append(int(r))
        return r

    _backward = torch.Tensor.backward

    def backward(self, *a, **k):
        if self.dim() == 0 and not rec.get("in_raster"):
            rec["loss"].append(float(self.detach()))
        return _backward(self, *a, **k)

    torch.optim.Adam = RecordingAdam
    importlib.import_module("torch._dynamo")   # Adam's step imports it; its import scan cannot see the stand-ins
    from avatarclip_b200 import conf as conf_mod
    pyhocon = types.ModuleType("pyhocon")
    pyhocon.ConfigFactory = types.SimpleNamespace(parse_string=conf_mod.parse_string)
    sys.modules.update({"pyhocon": pyhocon, "clip": clip, "smplx": smplx, "human_body_prior": hbp,
                        "human_body_prior.tools": tools, "human_body_prior.tools.model_loader": loader,
                        "human_body_prior.models": models, "human_body_prior.models.vposer_model": vpm,
                        "neural_renderer": nr, "tqdm": tqdm, "visualize": visualize})

    cwd = os.getcwd()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data"))
        OS.write_uv_obj(os.path.join(tmp, "data"), tv, tf)
        tok_holder["tok"] = ClipTokenizer(OS.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        text_feature = oct.encode_text(text, tok_holder["tok"].tokenize(O.TEXT).long())[0]
        torch.save(O.make_codebook(text_feature.detach().float()), os.path.join(tmp, "data", "codebook.pth"))
        torch.save({"state_dict": vae_sd}, os.path.join(tmp, "data", "motion_vae.pth"))
        os.chdir(tmp)
        sys.path.insert(0, REF)
        np.random.randint = randint
        torch.Tensor.backward = backward
        try:
            import main as ref_main
            for name, kw in RUNS.items():
                for k in ("param", "grad", "st_idx", "elevation", "azimuth", "rows", "loss"):
                    rec[k] = []
                p = os.path.join(tmp, f"{name}.conf")
                with open(p, "w") as fp:
                    fp.write(f"general {{\n    base_exp_dir = {tmp}/exp_{name}\n    mode = motion\n    text = {O.TEXT}\n"
                             "}\n\npose_generator {\n    type = VPoserCodebook\n}\n\nmotion_generator {\n"
                             "    type = MotionOptimizer\n" + "".join(f"    {k} = {v}\n" for k, v in kw.items()) + "}\n")
                np.random.seed(NP_SEED)
                torch.manual_seed(TORCH_SEED)
                ref_main.main(p)
                d = f"{tmp}/exp_{name}"
                assert rec["azimuth"] == [150.0] * NUM_ITER and len(rec["st_idx"]) == NUM_ITER
                assert len(rec["loss"]) == NUM_ITER and len(rec["param"]) == NUM_ITER, (len(rec["loss"]), len(rec["param"]))
                out[name] = dict(latent_init=rec["init"], optim_cfg=rec["optim_cfg"],
                                 st_idx=torch.tensor(rec["st_idx"], dtype=torch.int32),
                                 elevation=torch.tensor(rec["elevation"], dtype=torch.float64),
                                 rows=torch.tensor(rec["rows"]), loss=torch.tensor(rec["loss"]),
                                 params=torch.stack(rec["param"]), grads=torch.stack(rec["grad"]),
                                 motion=torch.from_numpy(np.load(f"{d}/motion.npy")),
                                 poses=torch.stack([torch.from_numpy(np.load(f"{d}/candidate_{i}.npy"))
                                                    for i in range(5)]))
                out[name]["latent"] = rec["param_obj"].detach().clone()     # after the last step
                print(f"[pin_motion_clip] {name}: st_idx {rec['st_idx']}, elevations "
                      f"{[round(e, 4) for e in rec['elevation']]}, losses {rec['loss']}, |grad_0| max "
                      f"{float(out[name]['grads'][0].abs().max()):.3e}")
        finally:
            os.chdir(cwd)
            torch.Tensor.backward = _backward
            np.random.randint = _randint

    assert torch.equal(out["shipped"]["poses"], out["clip_only"]["poses"])
    rec_out = dict(text=O.TEXT, np_seed=NP_SEED, torch_seed=TORCH_SEED, num_iter=NUM_ITER,
                   seeds=dict(vposer=O.VPOSER_SEED, motion_vae=OM.MOTION_VAE_SEED, codebook=O.CODEBOOK_SEED),
                   text_feature=text_feature.detach().float(), poses=out["shipped"]["poses"],
                   conf={n: dict(recon_coef=kw.get("recon_coef", [1, 0.8, 0.6, 0.4, 0.2]),
                                 delta_coef=kw.get("delta_coef", 0.01), clip_coef=kw.get("clip_coef", 0.001),
                                 clip_num_part=30, lr=0.01) for n, kw in RUNS.items()},
                   runs={n: {k: v for k, v in r.items() if k != "poses"} for n, r in out.items()})
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(rec_out, os.path.join(GOLDEN, "ref_motion_clip_small.pt"))


if __name__ == "__main__":
    main()
