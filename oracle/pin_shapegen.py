"""Pin oracle/shapegen.py against the reference's own ShapeGen (AvatarGen/ShapeGen/main.py ``shape_gen``, utils.py
``writeOBJ`` / ``readOBJ``) run in THIS container on the CPU, and record what it computed as
tests/golden/ref_shapegen_small.pt.

main.py / utils.py import ``clip``, ``smplx``, ``neural_renderer``, ``imageio``, ``matplotlib`` and ``tqdm``, none of
which is installed.  This script puts stand-ins for them in ``sys.modules`` and imports the UNMODIFIED files:
  * ``clip``: ``load`` returns a perceptor whose ``encode_text`` / ``encode_image`` are the oracle CLIP towers
    (oracle/clip_text.py, oracle/clip_vit.py) with seeded random weights; ``tokenize`` is ``ClipTokenizer`` on a merges
    file without merges (one token per byte);
  * ``neural_renderer``: ``load_obj`` / ``Renderer(camera_mode='look_at')`` / ``get_points_from_angles`` are the
    oracle's texture loading and textured rasteriser (PARITY UNPINNED, see oracle/shapegen.py);
  * ``smplx.build_layer``: a holder of the template's ``v_template`` / ``faces``;
  * ``.cuda()``: the identity.
Inputs are synthetic and regenerated from the seeds of oracle/shapegen.py: full-size LinearVAE weights, the shipped
template (tests/golden/ref_tree_template.tar.gz) with a seeded UV obj + mtl + PNGs, a 48-entry codebook built around
the neutral embedding so that the winner leads the runner-up by >= 0.05.  The golden holds outputs, the codebook and
the seeds; the 1.4 GB of weights are regenerated.  Nothing of the reference is copied into this repository.

    python -m oracle.pin_shapegen
"""
import math
import os
import sys
import tempfile
import types

import numpy as np
import torch

REF = "/root/reference/AvatarGen/ShapeGen"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
PROMPTS = ["a 3d rendering of a person in unreal engine", "a tall man:2", "tall: broad:0.5:-3", "a:b:1:2", "x:1e-1",
           "time 10:30: 1:-inf", ":3"]


def _small_obj_mesh():
    rng = np.random.default_rng(3)
    v = (rng.normal(0, 1, (6, 3)) * [1e-3, 1.0, 3e4]).astype(np.float32)
    v[0, 0] = np.float32(0.1)
    f = np.array([[0, 1, 2], [2, 3, 4], [4, 5, 0]], dtype=np.int64)
    return v, f


def main():
    from oracle import clip_text as oct
    from oracle import clip_vit as ocv
    from oracle import drive as D
    from oracle import shapegen as O
    sys.path.insert(0, ROOT)
    from avatarclip_b200.clip_tokenizer import ClipTokenizer

    tv, tf = D.template_obj()
    vae = O.vae_state(tv)
    visual, text = O.clip_states()
    vis = {k[len("visual."):]: v for k, v in visual.items()}
    recorded = {}

    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data"))
        uv_obj = O.write_uv_obj(os.path.join(tmp, "data"), tv, tf)
        tok = ClipTokenizer(O.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        tex = O.load_obj_textures(uv_obj)
        eye = (2 * math.sin(math.radians(150)), 0.0, -2 * math.cos(math.radians(150)))

        # the oracle's pass, to build the codebook around e and delta
        v0 = O.vae_decode(torch.zeros(1, 16), vae["dec1.weight"], vae["dec1.bias"], vae["dec2.weight"],
                          vae["dec2.bias"], tv)
        img = O.raster_textured(v0.reshape(-1, 3), tf, tex, eye)
        prep = O.clip_prep_nearest(torch.from_numpy(img).float().permute(2, 0, 1)[None])
        e = ocv.encode_image(vis, prep).mean(0)
        enc = lambda s: oct.encode_text(text, tok.tokenize(s).long())
        ntxt, ttxt = O.NEUTRAL_TXT, O.TARGET_TXT.rsplit(":", 2)[0]
        delta = (enc(ttxt) - enc(ntxt)).squeeze(0)
        codebook = O.make_codebook(e, delta)
        (latents, emb), = codebook.items()
        cos = O.codebook_cos(emb, e, delta)
        order = np.argsort(-cos)
        assert order[0] == O.CODEBOOK_WINNER and cos[order[0]] - cos[order[1]] >= 0.05, cos[order[:2]]
        torch.save(vae, os.path.join(tmp, "data", "model_VAE_16.pth"))
        torch.save(codebook, os.path.join(tmp, "data", "codebook.pth"))

        # stand-ins
        torch.Tensor.cuda = lambda self, *a, **k: self
        torch.nn.Module.cuda = lambda self, *a, **k: self

        class Perceptor:
            def eval(self):
                return self

            def requires_grad_(self, flag=True):
                return self

            def cuda(self):
                return self

            def encode_text(self, tokens):
                return oct.encode_text(text, tokens.long())

            def encode_image(self, images):
                recorded["prep"] = images.clone()
                return ocv.encode_image(vis, images.float())

        clip = types.ModuleType("clip")
        clip.load = lambda name, jit=False: (Perceptor(), None)
        clip.tokenize = lambda s: tok.tokenize(s).long()

        class Renderer:
            def __init__(self, camera_mode="look_at", image_size=256):
                assert camera_mode == "look_at"
                self.image_size, self.eye = image_size, None

            def cuda(self):
                return self

            def __call__(self, vertices, faces, textures):
                imgs = [torch.from_numpy(O.raster_textured(vertices[b].double().numpy(), faces[b].numpy(),
                                                           textures[b].double().numpy(), self.eye, n=self.image_size))
                        for b in range(vertices.shape[0])]
                out = torch.stack(imgs).permute(0, 3, 1, 2).float()
                recorded.setdefault("renders", []).append((tuple(float(x) for x in self.eye), out))
                return out, None, None

        nr = types.ModuleType("neural_renderer")
        nr.load_obj = lambda fname, load_texture=True, texture_size=8: (
            None, None, torch.from_numpy(O.load_obj_textures(fname, texture_size)).float())
        nr.Renderer = Renderer
        nr.get_points_from_angles = lambda d, el, az: (d * math.cos(math.radians(el)) * math.sin(math.radians(az)),
                                                       d * math.sin(math.radians(el)),
                                                       -d * math.cos(math.radians(el)) * math.cos(math.radians(az)))
        smplx = types.ModuleType("smplx")
        layer = types.SimpleNamespace(v_template=torch.from_numpy(tv), faces=tf.astype(np.int64))
        layer.cuda = lambda: layer
        smplx.build_layer = lambda folder, model_type, **kw: layer
        smplx_lbs = types.ModuleType("smplx.lbs")
        smplx_lbs.batch_rodrigues = None
        smplx.lbs = smplx_lbs
        blank = lambda name: types.ModuleType(name)
        tqdm = blank("tqdm")
        tqdm.tqdm = lambda it, *a, **k: it
        mpl = blank("matplotlib")
        mpl.pyplot = blank("matplotlib.pyplot")
        sys.modules.update({"clip": clip, "neural_renderer": nr, "smplx": smplx, "smplx.lbs": smplx_lbs,
                            "imageio": blank("imageio"), "matplotlib": mpl, "matplotlib.pyplot": mpl.pyplot,
                            "tqdm": tqdm})
        cwd = os.getcwd()
        os.chdir(tmp)
        sys.path.insert(0, REF)
        try:
            import utils as ref_utils
            import main as ref_main
            v, f, zero_beta_v = ref_main.shape_gen({"model_folder": None, "model_type": "smpl", "gender": "neutral",
                                                    "num_betas": 10}, "./data/model_VAE_16.pth",
                                                   "./data/codebook.pth", O.NEUTRAL_TXT, O.TARGET_TXT)
            parse = {p: ref_main.parse_prompt(p) for p in PROMPTS}
            sv, sf = _small_obj_mesh()
            ref_utils.writeOBJ(os.path.join(tmp, "small.obj"), sv, sf)
            obj_text = open(os.path.join(tmp, "small.obj")).read()
            rv, rf, _, _ = ref_utils.readOBJ(os.path.join(tmp, "small.obj"))
        finally:
            os.chdir(cwd)

    neutral = [img for eye_, img in recorded["renders"] if abs(eye_[0] - eye[0]) < 1e-12][0]
    ref_e = ocv.encode_image(vis, recorded["prep"]).mean(0)
    ref_delta = (enc(ttxt) - enc(ntxt)).squeeze(0)
    ref_cos = O.codebook_cos(emb, ref_e, ref_delta)
    best = int(np.argmax(ref_cos))
    dec_best = O.vae_decode(latents[best], vae["dec1.weight"], vae["dec1.bias"], vae["dec2.weight"], vae["dec2.bias"],
                            tv).reshape(-1, 3)

    # the restatement against the reference
    e_img = np.abs(neutral[0].permute(1, 2, 0).numpy() - img).max()
    e_v = np.abs(dec_best - v).max()
    e_v0 = np.abs(v0.reshape(-1, 3) - zero_beta_v).max()
    e_prep = (prep - recorded["prep"]).abs().max().item()
    e_cos = np.abs(ref_cos - cos).max()
    print(f"[pin_shapegen] best {best} (built {O.CODEBOOK_WINNER}), margin {np.sort(ref_cos)[-1] - np.sort(ref_cos)[-2]:.3f}")
    print(f"[pin_shapegen] max abs err: render {e_img:.2e}, clip input {e_prep:.2e}, cos {e_cos:.2e}, "
          f"decode(best) {e_v:.2e}, decode(0) {e_v0:.2e}")
    assert best == O.CODEBOOK_WINNER and max(e_v, e_v0) <= 1e-4 and e_img <= 1e-5 and e_cos <= 1e-4
    assert np.array_equal(rv, sv) and rf == sf.tolist()

    rec = dict(seeds=dict(vae=O.VAE_SEED, codebook=O.CODEBOOK_SEED, uv=O.UV_SEED, clip=O.CLIP_SEED),
               neutral_txt=O.NEUTRAL_TXT, target_txt=O.TARGET_TXT,
               codebook_latents=latents, codebook_emb=emb, best=best, cos=torch.from_numpy(ref_cos),
               image_embed=ref_e, delta_embed=ref_delta, v=torch.from_numpy(np.asarray(v, dtype=np.float32)),
               zero_beta_v=torch.from_numpy(np.asarray(zero_beta_v, dtype=np.float32)),
               neutral_image=neutral[0].half(), small_obj=dict(v=torch.from_numpy(sv), f=torch.from_numpy(sf),
                                                               text=obj_text),
               parse_prompt=parse)
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(rec, os.path.join(GOLDEN, "ref_shapegen_small.pt"))


if __name__ == "__main__":
    main()
