"""Pin oracle/animate.py against the reference's own pose stage (AvatarAnimate/models/pose_generation.py, builder.py,
main.py) run in THIS container on the CPU, and record what it computed as tests/golden/ref_animate_small.pt.

pose_generation.py / render.py / main.py import ``clip``, ``smplx``, ``human_body_prior``, ``neural_renderer``,
``tqdm``, ``pyhocon`` and visualize.py's renderer, none of which is installed.  This script puts stand-ins for them in
``sys.modules`` and imports the UNMODIFIED files:
  * ``clip``: ``load`` returns the oracle CLIP towers (oracle/clip_text.py, oracle/clip_vit.py) with seeded weights,
    ``tokenize`` is ``ClipTokenizer`` on a merges file without merges;
  * ``smplx.create``: SMPL with zero betas through oracle/lbs.py's my_lbs on the shipped template with synthetic
    SMPL tensors (oracle/drive.py golden_smpl);
  * ``human_body_prior``: ``load_model`` returns oracle/animate.py's VPoser decoder on seeded weights (PARITY UNPINNED);
  * ``neural_renderer``: the oracle texture loading and textured rasteriser of oracle/shapegen.py (PARITY UNPINNED);
  * ``pyhocon``: avatarclip_b200/conf.py's reader; ``tqdm``; ``visualize`` (main.py's jpg writer): records the poses it is handed.
torch's ``"cuda"`` device is mapped to the CPU.  Both generators run from ``main.main`` on pose confs:
VPoserCodebook with its defaults on a seeded 256-entry codebook built around the text feature (distinct top-40
cosines, near-duplicate latents in the top-40 for the suppression), and VPoserRealNVP with topk 2, num_batch 2,
num_sample 3 passed through the conf.  The torch prior draws and the numpy elevation draws are recorded in the order
the reference made them.  Nothing of the reference is copied into this repository.

    python -m oracle.pin_animate
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
NP_SEED = 5
TORCH_SEED = 6
REALNVP_CONF = dict(topk=2, num_batch=2, num_sample=3)


def main():
    from oracle import animate as O
    from oracle import clip_text as oct
    from oracle import clip_vit as ocv
    from oracle import drive as D
    from oracle import shapegen as OS
    sys.path.insert(0, ROOT)
    from avatarclip_b200.clip_tokenizer import ClipTokenizer

    tv, tf = D.template_obj()
    smpl = D.golden_smpl()
    visual, text = OS.clip_states()
    vis = {k[len("visual."):]: v for k, v in visual.items()}
    vp_sd = O.vposer_state()
    nvp_sd = O.realnvp_state()
    rec = {"eyes": [], "z": [], "vposer_inputs": [], "cos": []}

    # ---- stand-ins
    _tto, _mto = torch.Tensor.to, torch.nn.Module.to
    cpu = lambda a: tuple("cpu" if (isinstance(x, str) and x.startswith("cuda")) else x for x in a)
    torch.Tensor.to = lambda self, *a, **k: _tto(self, *cpu(a), **{kk: ("cpu" if kk == "device" else v)
                                                                   for kk, v in k.items()})
    torch.nn.Module.to = lambda self, *a, **k: _mto(self, *cpu(a), **{kk: ("cpu" if kk == "device" else v)
                                                                      for kk, v in k.items()})
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

    class SMPLLayer(torch.nn.Module):
        faces = tf.astype(np.int64)

        def forward(self, body_pose, global_orient):
            v = O.smpl_vertices(smpl, body_pose, global_orient[0].tolist())
            return types.SimpleNamespace(vertices=torch.from_numpy(v).float())

    smplx = types.ModuleType("smplx")
    smplx.create = lambda path, model_type: SMPLLayer()

    class VPoser(torch.nn.Module):
        def decode(self, z):
            rec["vposer_inputs"].append(z.clone())
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

    class Renderer:
        def __init__(self, camera_mode="look_at", image_size=256):
            assert camera_mode == "look_at"
            self.image_size, self.eye = image_size, None

        def to(self, device):
            return self

        def __call__(self, vertices, faces, textures):
            rec["eyes"].append(tuple(float(x) for x in self.eye))
            imgs = [torch.from_numpy(OS.raster_textured(vertices[b].double().numpy(), faces[b].numpy(),
                                                        textures[b].double().numpy(), self.eye, n=self.image_size))
                    for b in range(vertices.shape[0])]
            return torch.stack(imgs).permute(0, 3, 1, 2).float(), None, None

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

    from torch import distributions
    _sample = distributions.MultivariateNormal.sample

    def sample(self, shape=torch.Size()):
        z = _sample(self, shape)
        rec["z"].append(z.clone())
        return z

    distributions.MultivariateNormal.sample = sample
    from avatarclip_b200 import conf as conf_mod
    pyhocon = types.ModuleType("pyhocon")
    pyhocon.ConfigFactory = types.SimpleNamespace(parse_string=conf_mod.parse_string)
    sys.modules.update({"pyhocon": pyhocon, "clip": clip, "smplx": smplx, "human_body_prior": hbp, "human_body_prior.tools": tools,
                        "human_body_prior.tools.model_loader": loader, "human_body_prior.models": models,
                        "human_body_prior.models.vposer_model": vpm, "neural_renderer": nr, "tqdm": tqdm,
                        "visualize": visualize})

    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data"))
        OS.write_uv_obj(os.path.join(tmp, "data"), tv, tf)
        tok_holder["tok"] = ClipTokenizer(OS.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        text_feature = oct.encode_text(text, tok_holder["tok"].tokenize(O.TEXT).long())[0]
        codebook = O.make_codebook(text_feature)
        torch.save(codebook, os.path.join(tmp, "data", "codebook.pth"))
        torch.save({"state_dict": nvp_sd}, os.path.join(tmp, "data", "pose_realnvp.pth"))
        confs = {}
        for name, extra in (("VPoserCodebook", ""), ("VPoserRealNVP", "\n".join(
                f"    {k} = {v}" for k, v in REALNVP_CONF.items()))):
            p = os.path.join(tmp, f"{name}.conf")
            with open(p, "w") as fp:
                fp.write(f"general {{\n    base_exp_dir = {tmp}/exp_{name}\n    mode = pose\n    text = {O.TEXT}\n}}\n\n"
                         f"pose_generator {{\n    type = {name}\n{extra}\n}}\n")
            confs[name] = p
        os.chdir(tmp)
        sys.path.insert(0, REF)
        try:
            import main as ref_main
            import models.pose_generation as ref_pg

            class RecordingF:       # torch.nn.functional with every cosine_similarity the generators compute recorded
                def __getattr__(self, name):
                    return getattr(torch.nn.functional, name)

                def cosine_similarity(self, *a, **k):
                    c = torch.nn.functional.cosine_similarity(*a, **k)
                    rec["cos"].append(c.detach().clone().reshape(-1))
                    return c

            ref_pg.F = RecordingF()
            out = {}
            for name in ("VPoserCodebook", "VPoserRealNVP"):
                for k in rec:
                    rec[k] = []
                np.random.seed(NP_SEED)
                torch.manual_seed(TORCH_SEED)
                try:
                    ref_main.main(confs[name])
                except SystemExit as e:
                    assert e.code == 0, e.code
                d = f"{tmp}/exp_{name}"
                out[name] = dict(poses=torch.stack([torch.from_numpy(np.load(f"{d}/candidate_{i}.npy"))
                                                    for i in range(len([f for f in os.listdir(d) if f.endswith(".npy")]))]),
                                 eyes=torch.tensor(rec["eyes"]), z=[z.clone() for z in rec["z"]],
                                 vposer_inputs=[z.clone() for z in rec["vposer_inputs"]],
                                 cos=[c.clone() for c in rec["cos"]])
        finally:
            os.chdir(cwd)

    # ---- the restatement against the reference
    cb = out["VPoserCodebook"]
    cos = O.cosine(codebook["codebook_embedding"], text_feature)
    top = np.argsort(-cos, kind="stable")[:40]
    poses40, _ = O.vposer_decode(codebook["codebook"][top], vp_sd)
    keep = O.suppress(poses40.reshape(40, -1), 0.07)[:5]
    e_cb = np.abs(poses40.reshape(40, -1)[keep] - cb["poses"].double().numpy()).max()
    srt = np.sort(cos)[::-1]
    print(f"[pin_animate] codebook: kept {keep}, top-41 gap {np.min(srt[:40] - srt[1:41]):.4f}, pose err {e_cb:.2e}")
    P = poses40.reshape(40, -1).astype(np.float32)
    md = [min(np.abs(P[i] - P[j]).astype(np.float64).mean() for j in O.suppress(P[:i], 0.07)) for i in range(1, 40)]
    print(f"[pin_animate] codebook: greedy distances below the threshold <= {max(d for d in md if d <= 0.07):.4f}, "
          f"above >= {min(d for d in md if d > 0.07):.4f}")
    assert all(d < 0.01 or d > 0.1 for d in md)
    assert len(keep) == 5 and e_cb <= 1e-5 and len(set(keep)) == 5 and max(keep) < 40 and keep != list(range(5))

    nv = out["VPoserRealNVP"]
    zs = torch.cat(nv["z"]).reshape(REALNVP_CONF["topk"], -1, 32)
    x = O.realnvp_decode(zs[0], text_feature, nvp_sd)
    e_x = np.abs(x - torch.cat(nv["vposer_inputs"][:REALNVP_CONF["num_batch"]]).double().numpy()).max()
    print(f"[pin_animate] realnvp: {len(nv['z'])} prior draws, {len(nv['eyes'])} renders, decode err {e_x:.2e}")
    assert e_x <= 1e-4 and len(nv["eyes"]) == 5 * (REALNVP_CONF["topk"] * REALNVP_CONF["num_batch"] +
                                                     REALNVP_CONF["topk"])

    # the reference's cosines: per candidate one [num_sample] call per batch, then one [1] call per candidate in the sort
    K, nb, ns = REALNVP_CONF["topk"], REALNVP_CONF["num_batch"], REALNVP_CONF["num_sample"]
    assert len(nv["cos"]) == K * nb + K and all(c.numel() == ns for c in nv["cos"][:K * nb])
    scores = torch.stack([torch.cat(nv["cos"][k * nb:(k + 1) * nb]) for k in range(K)])
    sort_scores = torch.cat(nv["cos"][K * nb:])
    best_scores = []
    for k in range(K):                 # get_pose's running best, from 0
        b = 0.0
        for g in range(nb):
            m = float(scores[k, g * ns:(g + 1) * ns].max())
            b = m if m > b else b
        best_scores.append(b)
    best_scores = torch.tensor(best_scores)

    rec_out = dict(text=O.TEXT, np_seed=NP_SEED, torch_seed=TORCH_SEED,
                   seeds=dict(vposer=O.VPOSER_SEED, realnvp=O.REALNVP_SEED, codebook=O.CODEBOOK_SEED,
                              clip=OS.CLIP_SEED, uv=OS.UV_SEED),
                   realnvp_conf=REALNVP_CONF, text_feature=text_feature.float(),
                   codebook=dict(topk=torch.from_numpy(top.copy()), keep=torch.tensor(keep), poses=cb["poses"],
                                 cos=torch.from_numpy(cos)),
                   realnvp=dict(z=zs, eyes=nv["eyes"], poses=nv["poses"], scores=scores, best_scores=best_scores,
                                sort_scores=sort_scores))
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(rec_out, os.path.join(GOLDEN, "ref_animate_small.pt"))


if __name__ == "__main__":
    main()
