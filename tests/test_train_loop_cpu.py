"""Runner.train (--mode train, the NeuS pre-fit) against the reference's own loop text (main.py:180-256 + :568-586) executed in
place on the CPU: same fake dataset (random pixel batches from torch's global generator), same differentiable fake renderer
over the network parameters, `torch.optim.Adam`, identical seeds.  Pins the loop's host logic -- image permutation cycling,
mask handling, the loss formula, optimiser stepping, WHEN the learning rate is updated, what is logged under which name -- not
the renderer (GPU parity tests).  What the reference's lines produced is stored under tests/golden/
(util_neus.reference_golden)."""
import copy
import os
import textwrap
import types

import pytest
import torch
import torch.nn.functional as F

from util_neus import reference_golden

REF_MAIN = os.path.join(os.environ.get("AVC_REFERENCE", ""), "AvatarGen/AppearanceGen/main.py")
HERE = os.path.dirname(os.path.abspath(__file__))


class FakeDataset:
    n_images, H, W = 5, 16, 16

    def __init__(self):
        g = torch.Generator().manual_seed(1)
        self.images = torch.rand(5, 16, 16, 3, generator=g)
        self.masks = (torch.rand(5, 16, 16, 1, generator=g) > 0.4).float() * torch.rand(5, 16, 16, 1, generator=g)

    def gen_random_rays_at(self, img_idx, batch_size):
        img_idx = int(img_idx)
        px = torch.randint(low=0, high=self.W, size=[batch_size])
        py = torch.randint(low=0, high=self.H, size=[batch_size])
        d = torch.stack([(px - 8.0) / 16, -(py - 8.0) / 16, -torch.ones(batch_size)], -1)
        d = d / d.norm(dim=-1, keepdim=True)
        o = torch.tensor([0.1 * img_idx, 0.0, 1.5]).expand(batch_size, 3)
        return torch.cat([o, d, self.images[img_idx][(py, px)], self.masks[img_idx][(py, px)]], -1)

    def near_far_from_sphere(self, o, d, is_sphere=False):
        return torch.zeros(o.shape[0], 1), torch.ones(o.shape[0], 1) * 2


def make_render(params):
    def render(rays_o, rays_d, near, far, background_rgb=None, cos_anneal_ratio=0.0, **kw):
        s = sum((p * p).sum() for p in params) * 1e-4 + sum(p.sum() for p in params) * 1e-3
        wsum = torch.sigmoid(rays_o[:, :1] * s + rays_d[:, 1:2] * 3)
        return {"color_fine": torch.sigmoid(rays_d * 2 + s), "s_val": wsum * 0.1 + s, "cdf_fine": wsum.expand(-1, 4) * 0.5,
                "gradient_error": (s - 0.3) ** 2, "weight_max": wsum * 0.5, "weight_sum": wsum, "extra_color_fine": None}
    return render


class Writer:
    def __init__(self):
        self.rec = []

    def add_scalar(self, name, value, step):
        self.rec.append((name, float(value), int(step)))


def _reference_methods():
    lines = open(REF_MAIN).read().split("\n")
    assert lines[179].strip() == "def train(self):" and "image_perm = self.get_image_perm()" in lines[255]
    assert lines[567].strip() == "def get_image_perm(self):" and "g['lr']" in lines[585]
    ns = dict(np=__import__("numpy"), torch=torch, F=F, os=os, tqdm=lambda it: it)
    exec(textwrap.dedent("\n".join(lines[179:256])), ns)
    exec(textwrap.dedent("\n".join(lines[567:586])), ns)
    return ns


@pytest.mark.parametrize("mask_weight,white", [(0.5, False), (0.0, True)])
def test_mode_train_loop_equals_the_reference_loop(tmp_path, mask_weight, white, capsys):
    from avatarclip_b200.runner import Runner
    conf = open(os.path.join(HERE, "runner_conf_sample.conf")).read().replace("./exp/CASE_NAME/demo", str(tmp_path / "ours"))
    for old, new in (("end_iter = 100000", "end_iter = 12"), ("warm_up_end = 500", "warm_up_end = 4"), ("batch_size = 512", "batch_size = 40"),
                     ("mask_weight = 0.5", f"mask_weight = {mask_weight}"), ("use_white_bkgd = False", f"use_white_bkgd = {white}"),
                     ("report_freq = 100", "report_freq = 3")):
        assert old in conf
        conf = conf.replace(old, new)
    p = tmp_path / "c.conf"
    p.write_text(conf)
    r = Runner(str(p), mode="train", case="smpl", device="cpu")
    r.dataset = FakeDataset()

    def reference():
        # independent copies of the same networks, torch.optim.Adam over sdf + variance + colour (main.py:141-145)
        nets = [copy.deepcopy(m) for m in (r.sdf_network, r.deviation_network, r.color_network)]
        ref_params = [q for m in nets for q in m.parameters()]
        ns = _reference_methods()
        wr_ref = Writer()
        ns["SummaryWriter"] = lambda log_dir=None: wr_ref
        ref = types.SimpleNamespace(
            base_exp_dir=str(tmp_path / "ref"), end_iter=12, iter_step=0, dataset=FakeDataset(), batch_size=40, use_white_bkgd=white,
            mask_weight=mask_weight, igr_weight=r.igr_weight, report_freq=3, save_freq=10 ** 9, val_freq=10 ** 9, val_mesh_freq=10 ** 9,
            warm_up_end=4.0, anneal_end=0.0, learning_rate=r.learning_rate, learning_rate_alpha=r.learning_rate_alpha,
            renderer=types.SimpleNamespace(render=make_render(ref_params)), optimizer=torch.optim.Adam(ref_params, lr=r.learning_rate))
        for name in ("get_image_perm", "get_cos_anneal_ratio", "update_learning_rate"):
            setattr(ref, name, types.MethodType(ns[name], ref))
        torch.manual_seed(7)
        ns["train"](ref)
        return dict(rec=wr_ref.rec, params=[q.detach() for q in ref_params], lr=ref.optimizer.param_groups[0]["lr"],
                    out=capsys.readouterr().out, iter_step=ref.iter_step)
    want = reference_golden(f"mode_train_{mask_weight}_{white}", reference)
    wr_ref, ref_params, ref_out = types.SimpleNamespace(rec=want["rec"]), want["params"], want["out"]
    # our side
    wr = Writer()
    r._make_writer = lambda: wr
    r.save_freq = r.val_freq = r.val_mesh_freq = 10 ** 9
    r.renderer.render = make_render(r._all_params())
    torch.manual_seed(7)
    logs = []
    assert r.train(log=logs.append, validate=False) == 12 == want["iter_step"]
    assert [n for n, _, _ in wr.rec] == [n for n, _, _ in wr_ref.rec]                # same scalar names in the same order
    assert [s for _, _, s in wr.rec] == [s for _, _, s in wr_ref.rec]
    worst = max(abs(a - b) / max(abs(b), 1e-12) for (_, a, _), (_, b, _) in zip(wr.rec, wr_ref.rec))
    assert worst < 1e-6, worst
    for a, b in zip(r._all_params(), ref_params):                                    # the same parameters after 12 Adam steps
        assert torch.allclose(a.detach(), b.detach(), rtol=1e-6, atol=1e-9)
    assert r.optimizer.param_groups[0]["lr"] == want["lr"]
    lr_ours = [str(m).split("lr=")[1] for m in logs if "lr=" in str(m)]
    lr_ref = [l.split("lr=")[1] for l in ref_out.splitlines() if "lr=" in l]
    assert lr_ours == lr_ref and len(lr_ours) == 4                                   # the lr in force at steps 3, 6, 9, 12


def test_train_clip_host_logic_equals_the_reference_lines(tmp_path, monkeypatch):
    """What Runner.train_clip hands to the fused step, step by step -- camera pose, background mode, light, ambience (numpy's
    global stream seeded by train.seed), WHICH cached text embedding (main.py:499-507: face every 4th step, back when the camera
    is behind, else body), the learning rate in force (update_learning_rate before the loop and after every step, :339,563)
    and the cosine-anneal ratio -- against the reference's own lines executed in place.  The step itself is mocked (GPU tests)."""
    import numpy as np
    from avatarclip_b200 import views
    from avatarclip_b200.runner import Runner
    conf = open(os.path.join(HERE, "runner_conf_sample.conf")).read().replace("./exp/CASE_NAME/demo", str(tmp_path / "ours"))
    conf = conf.replace("warm_up_end = 500", "warm_up_end = 5").replace("end_iter = 100000", "end_iter = 80")
    p = tmp_path / "c.conf"
    p.write_text(conf)
    r = Runner(str(p), mode="train_clip", case="smpl", device="cpu")                  # seeds numpy with train.seed = 11
    n_steps = 48
    body, face, back = torch.zeros(1, 4), torch.ones(1, 4), torch.full((1, 4), 2.0)
    r.encoded_text, r.encoded_face_text, r.encoded_back_text = body, face, back
    r.clip_tower, r.v, r.f = object(), torch.zeros(1, 3, 3), np.zeros((1, 3), dtype=np.int64)
    r.dataset = types.SimpleNamespace(H=256, W=256, focal=221.7, n_images=0)
    rec = []

    class FakeTrainer:
        iter_step, scalars, cos, _out = 0, None, None, None

        def set_text(self, emb):
            self.text = emb

        def step(self, view, lr=None, cos_anneal=1.0):
            d = view.draw
            rec.append(dict(text=float(self.text[0, 0]), lr=lr, cos_anneal=cos_anneal, pose=d.pose.copy(), bg=d.bg_choice,
                            light=d.light_dir.copy(), ambience=d.ambience, face=d.face_step, is_front=d.is_front))
            return torch.tensor(1.0)

    class FakeBuilder:
        def __init__(self, *a, **k):
            pass

        def submit(self, draw):
            return draw

        def finish(self, pending):
            return types.SimpleNamespace(draw=pending)

    r.trainer = FakeTrainer()
    monkeypatch.setattr(views, "ViewBuilder", FakeBuilder)
    r._make_writer = lambda: __import__("avatarclip_b200.runner", fromlist=["_NullWriter"])._NullWriter()
    assert r.train_clip(max_steps=n_steps, log=lambda m: None, validate=False) == n_steps
    # ---- the reference's lines

    def reference():
        from oracle.pin_loss_stage import cut
        from oracle.pin_sampling import reference_draws
        ref = reference_draws(r.seed, n_steps + 1, r.head_height, face=True, bg_aug=True, shading=True)   # ours looks one step ahead
        prompt_lines = cut("main.py", 499, 507, "if self.use_face_prompt and iter_i % 4 == 0", "current_no_texture_text_encoding = self.encoded_text")
        sched = {"np": np}
        exec(cut("main.py", 571, 586, "def get_cos_anneal_ratio", "g['lr']"), sched)
        out = []
        for i in range(n_steps):
            s = types.SimpleNamespace(use_face_prompt=True, use_back_prompt=True, encoded_text=body, encoded_face_text=face,
                                      encoded_back_text=back)
            loc = dict(self=s, iter_i=i, is_front=ref[i]["is_front"])
            exec(prompt_lines, loc)
            sch = types.SimpleNamespace(iter_step=i, warm_up_end=5.0, end_iter=80, learning_rate_alpha=r.learning_rate_alpha,
                                        learning_rate=r.learning_rate, anneal_end=0.0,
                                        optimizer=types.SimpleNamespace(param_groups=[{"lr": None}]))
            sched["update_learning_rate"](sch)
            out.append(dict(text=float(loc["current_text_encoding"][0, 0]), no_texture=float(loc["current_no_texture_text_encoding"][0, 0]),
                            lr=sch.optimizer.param_groups[0]["lr"], cos_anneal=float(sched["get_cos_anneal_ratio"](sch)),
                            pose=np.asarray(ref[i]["pose"]), bg=ref[i]["choice_i"], light=np.asarray(ref[i]["light_dir"]).astype(np.float32),
                            ambience=ref[i]["ambience"]))
        return out
    want = reference_golden("train_clip_host_logic", reference)
    assert len(rec) == len(want) == n_steps
    for i, (got, w) in enumerate(zip(rec, want)):
        assert got["text"] == w["text"] == w["no_texture"], i
        assert got["lr"] == w["lr"], i
        assert got["cos_anneal"] == w["cos_anneal"]
        assert np.array_equal(got["pose"], w["pose"]) and got["bg"] == w["bg"], i
        assert np.array_equal(got["light"], w["light"]) and got["ambience"] == w["ambience"]
    assert {g["text"] for g in rec} == {0.0, 1.0, 2.0}             # body, face and back prompts all occurred
