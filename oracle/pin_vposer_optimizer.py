"""Pin AvatarAnimate's VPoserOptimizer loop against the reference's own code (AvatarAnimate/models/pose_generation.py,
builder.py, main.py) run in THIS container on the CPU, and record what it computed as
tests/golden/ref_vposer_optimizer_small.pt.

The stand-ins are oracle/pin_pose_optimizer.py's (SMPL through fp64 autograd of my_lbs, the textured render with the
oracle's restatement of neural_renderer's backward, the oracle CLIP towers, pyhocon, tqdm, visualize), with one
addition: ``human_body_prior.tools.model_loader.load_model`` returns oracle/vposer_optimizer.py's VPoserDecoder on
oracle/animate.py's ``vposer_state()`` weights, an fp64 autograd restatement of VPoser's decode.  torch's ``"cuda"``
device is mapped to the CPU, and ``torch.optim.Adam`` records each step's latent and gradient.  main.main runs a
VPoserOptimizer conf with topk 2 and num_iteration 3.

What this pins: the loop of the reference's own code -- the torch.randn(32) latent draws, the numpy elevation draws (5
per get_pose_feature call, candidate k's iterations before candidate k + 1's, then the sort's), the Adam steps and their
lr, the loss, the returned pose (the decode of the latent before the last step), pose_padding, the sort and the written
files.  What it does not pin: VPoser and torchgeometry themselves (``human_body_prior`` is absent, so the decoder is
this project's restatement, PARITY UNPINNED as oracle/animate.py states) and the rasteriser's gradient (neural_renderer
is absent); the recorded gradients are only as right as those restatements.  Nothing of the reference is copied into
this repository.

    python -m oracle.pin_vposer_optimizer
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
CONF = dict(topk=2, num_iteration=3)


def main():
    from oracle import animate as O
    from oracle import clip_text as oct
    from oracle import clip_vit as ocv
    from oracle import drive as D
    from oracle import lbs as olbs
    from oracle import pose_optimizer as OP
    from oracle import shapegen as OS
    from oracle import vposer_optimizer as OV
    sys.path.insert(0, ROOT)
    from avatarclip_b200.clip_tokenizer import ClipTokenizer

    tv, tf = D.template_obj()
    smpl = D.golden_smpl()
    visual, text = OS.clip_states()
    vis = {k[len("visual."):]: v for k, v in visual.items()}
    rec = {"eyes": [], "cos": [], "param": [], "grad": []}

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

    hbp = types.ModuleType("human_body_prior")
    tools = types.ModuleType("human_body_prior.tools")
    loader = types.ModuleType("human_body_prior.tools.model_loader")
    loader.load_model = lambda path, model_code=None, remove_words_in_model_weights=None, disable_grad=False: (
        OV.VPoserDecoder(O.vposer_state()), None)
    models = types.ModuleType("human_body_prior.models")
    vpm = types.ModuleType("human_body_prior.models.vposer_model")
    vpm.VPoser = torch.nn.Module

    class RasterFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, vertices, faces, textures, eye, n):
            v = vertices.detach().double().numpy()
            imgs, maps = [], []
            for b in range(v.shape[0]):
                if ctx.needs_input_grad[0]:
                    rgb, fidx, rgb_ss, proj = OP.raster_maps(v[b], faces[b].numpy(), textures[b].double().numpy(),
                                                             eye, n)
                    maps.append((fidx, rgb_ss, proj))
                else:
                    rgb = OS.raster_textured(v[b], faces[b].numpy(), textures[b].double().numpy(), eye, n=n)
                imgs.append(torch.from_numpy(rgb))
            ctx.save = (v, faces[0].numpy(), eye, maps)
            return torch.stack(imgs).permute(0, 3, 1, 2).float()

        @staticmethod
        def backward(ctx, g):
            v, faces, eye, maps = ctx.save
            e, rot = OS.look_at_camera(eye)
            gv = np.stack([OP.raster_backward_image(v[b], faces, proj, e, rot, fidx, rgb_ss,
                                                    g[b].permute(1, 2, 0).double().numpy(), 2)
                           for b, (fidx, rgb_ss, proj) in enumerate(maps)])
            return torch.from_numpy(gv).float(), None, None, None, None

    class Renderer:
        def __init__(self, camera_mode="look_at", image_size=256):
            assert camera_mode == "look_at"
            self.image_size, self.eye = image_size, None

        def to(self, device):
            return self

        def __call__(self, vertices, faces, textures):
            rec["eyes"].append(tuple(float(x) for x in self.eye))
            return RasterFn.apply(vertices, faces, textures, np.asarray(self.eye, dtype=np.float64),
                                  self.image_size), None, None

    nr = types.ModuleType("neural_renderer")
    nr.load_obj = lambda fname, load_texture=True, texture_size=8: (
        None, None, torch.from_numpy(OS.load_obj_textures(fname, texture_size)).float())
    nr.Renderer = Renderer
    nr.get_points_from_angles = lambda d, el, az: O.eye(el, az)
    tqdm = types.ModuleType("tqdm")
    tqdm.tqdm = lambda it, *a, **k: it
    visualize = types.ModuleType("visualize")
    visualize.render_pose = lambda pose, path: None
    visualize.render_motion = lambda motion, path: None

    class RecordingAdam(torch.optim.Adam):
        def step(self, closure=None):
            p = self.param_groups[0]["params"][0]
            rec["param"].append(p.detach().clone())
            rec["grad"].append(p.grad.detach().clone())
            torch.cuda.is_available = _avail        # the step itself runs torch's CPU Adam
            try:
                return super().step(closure)
            finally:
                torch.cuda.is_available = lambda: True

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
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data"))
        OS.write_uv_obj(os.path.join(tmp, "data"), tv, tf)
        tok_holder["tok"] = ClipTokenizer(OS.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        text_feature = oct.encode_text(text, tok_holder["tok"].tokenize(O.TEXT).long())[0]
        p = os.path.join(tmp, "po.conf")
        with open(p, "w") as fp:
            fp.write(f"general {{\n    base_exp_dir = {tmp}/exp\n    mode = pose\n    text = {O.TEXT}\n}}\n\n"
                     "pose_generator {\n    type = VPoserOptimizer\n" +
                     "".join(f"    {k} = {v}\n" for k, v in CONF.items()) + "}\n")
        os.chdir(tmp)
        sys.path.insert(0, REF)
        try:
            import main as ref_main
            import models.pose_generation as ref_pg

            class RecordingF:
                def __getattr__(self, name):
                    return getattr(torch.nn.functional, name)

                def cosine_similarity(self, *a, **k):
                    c = torch.nn.functional.cosine_similarity(*a, **k)
                    rec["cos"].append(c.detach().clone().reshape(-1))
                    return c

            ref_pg.F = RecordingF()
            np.random.seed(NP_SEED)
            torch.manual_seed(TORCH_SEED)
            try:
                ref_main.main(p)
            except SystemExit as e:
                assert e.code == 0, e.code
            files = [np.load(f"{tmp}/exp/candidate_{i}.npy") for i in range(CONF["topk"])]
        finally:
            os.chdir(cwd)

    K, T = CONF["topk"], CONF["num_iteration"]
    cos = torch.cat(rec["cos"])
    assert cos.numel() == K * T + K and len(rec["param"]) == K * T
    eyes = torch.tensor(rec["eyes"]).reshape(-1, 5, 3)
    assert eyes.shape[0] == K * T + K
    latents = torch.stack(rec["param"]).reshape(K, T, 32)
    # the returned pose is the decode of the latent before the last step
    poses = OV.decode(latents[:, -1].double(), O.vposer_state()).reshape(K, 63).float()
    out = dict(text=O.TEXT, np_seed=NP_SEED, torch_seed=TORCH_SEED, conf=CONF, text_feature=text_feature.float(),
               init=latents[:, 0].clone(), eyes=eyes, loss=(1 - cos[:K * T]).reshape(K, T), latents=latents,
               grads=torch.stack(rec["grad"]).reshape(K, T, 32), poses=poses, sort_scores=cos[K * T:],
               files=torch.from_numpy(np.stack(files)))
    print(f"[pin_vposer_optimizer] losses {out['loss'].tolist()}, sort scores {out['sort_scores'].tolist()}, "
          f"|grad| max {float(out['grads'].abs().max()):.3e}")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(out, os.path.join(GOLDEN, "ref_vposer_optimizer_small.pt"))


if __name__ == "__main__":
    main()
