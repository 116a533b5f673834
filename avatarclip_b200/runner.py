"""Host-side mirror of ``Runner`` (AvatarGen/AppearanceGen/main.py:30-945): same constructor arguments, conf keys,
checkpoint file layout (``sdf_network_fine`` / ``variance_network_fine`` / ``color_network_fine`` / ``optimizer`` /
``iter_step``), output file names and CLI flags (main.py:953-975) as the reference, over libavc_b200.so:

* ``train_clip``  (main.py:337-566) -- the hot path: per-step draws (``sampling.StepSampler``), view preparation on the
  device with one-step lookahead (``views.ViewBuilder``: template rasteriser, dilation, canvas, rays, targets,
  backgrounds), the fused step (``trainer.AppearanceTrainer``), face / back prompt selection, LR schedule, logging,
  checkpoints, periodic ``validate_image`` / ``validate_mesh``.
* ``train``       (main.py:180-256) -- NeuS pre-fit on the rendered template views (random-pixel batches, L1 + eikonal
  + BCE) through the differentiable ``NeuSRenderer.render`` seam and ``torch.optim.Adam``, as the reference.
* ``validate_image`` / ``validate_mesh`` / ``render_geometry_cast_light`` (main.py:634-919).

Without the ``clip`` package, ``init_clip`` encodes the conf's prompts itself from openai's ``ViT-B-32.pt`` and BPE
merges file (``clip_tokenizer`` / ``clip_text``).  Not importable here and therefore injected: ``smplx`` (pass template
vertices / faces, or the SMPL tensors, to ``init_smpl``).
"""
from __future__ import annotations

import argparse
import logging
import os
import random
from shutil import copyfile
from typing import Optional

import numpy as np
import torch

from . import conf as hocon
from .dataset import SMPL_Dataset
from .fields import RenderingNetwork, SDFNetwork, SingleVarianceNetwork
from .renderer import NeuSRenderer
from .sampling import StepSampler, lookat, sphere_coord


def _clip_importable() -> bool:
    try:
        import clip  # noqa: F401 (optional dependency)
    except ImportError:
        return False
    return True


def to8b(x):
    return (255 * np.clip(x, 0, 1)).astype(np.uint8)


class _NullWriter:
    def add_scalar(self, *a, **k):
        pass


class Runner:
    def __init__(self, conf_path, mode="train", case="CASE_NAME", is_continue=False, is_colab=False, conf=None,
                 device="cuda", engine: int = 1):
        self.device = torch.device(device)
        self.conf_path = conf_path
        if is_colab:
            self.conf = conf
        else:
            with open(self.conf_path) as f:
                conf_text = f.read().replace("CASE_NAME", case)
            self.conf = hocon.parse_string(conf_text)
        c = self.conf
        self.base_exp_dir = c["general.base_exp_dir"]
        os.makedirs(self.base_exp_dir, exist_ok=True)
        self.dataset = SMPL_Dataset(c["dataset"], device=self.device) if self.device.type == "cuda" else None
        self.iter_step = 0
        # training parameters (main.py:49-64)
        self.end_iter = c.get_int("train.end_iter")
        self.save_freq = c.get_int("train.save_freq")
        self.report_freq = c.get_int("train.report_freq")
        self.val_freq = c.get_int("train.val_freq")
        self.val_mesh_freq = c.get_int("train.val_mesh_freq", default=10 ** 9)
        self.batch_size = c.get_int("train.batch_size")
        self.validate_resolution_level = c.get_int("train.validate_resolution_level", default=1)
        self.learning_rate = c.get_float("train.learning_rate")
        self.learning_rate_alpha = c.get_float("train.learning_rate_alpha")
        self.use_white_bkgd = c.get_bool("train.use_white_bkgd", default=False)
        self.warm_up_end = c.get_float("train.warm_up_end", default=0.0)
        self.anneal_end = c.get_float("train.anneal_end", default=0.0)
        self.max_ray_num = c.get_int("train.max_ray_num", default=112 * 112)
        self.igr_weight = c.get_float("train.igr_weight")
        self.mask_weight = c.get_float("train.mask_weight")
        self.clip_weight = c.get_float("train.clip_weight", default=None)
        self.extra_color = c.get_bool("model.rendering_network.extra_color", default=False)
        self.add_no_texture = c.get_bool("train.add_no_texture", default=False)
        self.texture_cast_light = c.get_bool("train.texture_cast_light", default=False)
        self.use_face_prompt = c.get_bool("train.use_face_prompt", default=False)
        self.use_back_prompt = c.get_bool("train.use_back_prompt", default=False)
        self.use_silhouettes = c.get_bool("train.use_silhouettes", default=False)
        self.head_height = c.get_float("train.head_height", default=0.65)
        self.use_bg_aug = c.get_bool("train.use_bg_aug", default=True)
        self.seed = c.get_int("train.seed", default=None)
        if self.seed is not None:                                        # main.py:104-114
            torch.manual_seed(self.seed)
            if torch.cuda.is_available():
                torch.cuda.manual_seed_all(self.seed)
            random.seed(self.seed)
            np.random.seed(self.seed)
        self.smpl_model_path = c.get_string("general.smpl_model_path", default="../../smpl_models")
        self.pose_type = c.get_string("general.pose_type", default="stand_pose")
        self.is_continue, self.mode = is_continue, mode
        self.writer = None
        # networks (main.py:134-151): the conf subtrees are the constructor kwargs
        self.nerf_outside = None
        self.sdf_network = SDFNetwork(**c["model.sdf_network"]).to(self.device)
        self.deviation_network = SingleVarianceNetwork(**c["model.variance_network"]).to(self.device)
        self.color_network = RenderingNetwork(**c["model.rendering_network"]).to(self.device)
        self.renderer = NeuSRenderer(self.nerf_outside, self.sdf_network, self.deviation_network, self.color_network,
                                     engine=engine, **c["model.neus_renderer"])
        self.optimizer = None            # torch.optim.Adam of --mode train (built on first use)
        self.trainer = None              # fused step of --mode train_clip
        self.clip_tower = None
        self.encoded_text = self.encoded_face_text = self.encoded_back_text = None
        self.v = self.f = None
        self._pending_optimizer_state = None
        self.process_group, self.rank, self.world = None, 0, 1      # view-sharded multi-GPU: set_process_group()
        pretrain = c.get_string("train.pretrain", default=None)
        if pretrain is not None and os.path.exists(pretrain):
            logging.info("Load pretrain: %s", pretrain)
            self.load_pretrain(pretrain)
        elif pretrain is not None:
            logging.warning("train.pretrain = %s does not exist: starting from the geometric initialisation", pretrain)
        if is_continue:
            ckdir = os.path.join(self.base_exp_dir, "checkpoints")
            names = sorted(n for n in os.listdir(ckdir) if n.endswith("pth") and int(n[5:-4]) <= self.end_iter)
            if names:
                logging.info("Find checkpoint: %s", names[-1])
                self.load_checkpoint(names[-1])
        if self.mode[:5] == "train":
            self.file_backup()

    # ------------------------------------------------------------------ schedules (main.py:571-586)
    def get_image_perm(self):
        """main.py:568-569."""
        return torch.randperm(self.dataset.n_images)

    def get_cos_anneal_ratio(self):
        return 1.0 if self.anneal_end == 0.0 else float(np.min([1.0, self.iter_step / self.anneal_end]))

    def current_lr(self) -> float:
        if self.iter_step < self.warm_up_end:
            f = self.iter_step / self.warm_up_end
        else:
            a = self.learning_rate_alpha
            progress = (self.iter_step - self.warm_up_end) / (self.end_iter - self.warm_up_end)
            f = (np.cos(np.pi * progress) + 1.0) * 0.5 * (1 - a) + a
        return float(self.learning_rate * f)

    def update_learning_rate(self):
        if self.optimizer is not None:
            for g in self.optimizer.param_groups:
                g["lr"] = self.current_lr()

    def file_backup(self):
        """main.py:588-599: copy the conf (and the recorded source directories when they exist) next to the run."""
        rec = os.path.join(self.base_exp_dir, "recording")
        try:
            os.makedirs(rec, exist_ok=True)
            for dir_name in self.conf.get("general.recording", default=[]) or []:
                if not os.path.isdir(dir_name):
                    continue
                cur = os.path.join(rec, dir_name)
                os.makedirs(cur, exist_ok=True)
                for f_name in os.listdir(dir_name):
                    if f_name[-3:] == ".py":
                        copyfile(os.path.join(dir_name, f_name), os.path.join(cur, f_name))
            if self.conf_path and os.path.exists(self.conf_path):
                copyfile(self.conf_path, os.path.join(rec, "config.conf"))
        except OSError as e:
            logging.warning("file_backup: %s", e)

    def _make_writer(self):
        try:
            from torch.utils.tensorboard import SummaryWriter
            return SummaryWriter(log_dir=os.path.join(self.base_exp_dir, "logs"))
        except Exception:
            return _NullWriter()

    # ------------------------------------------------------------------ CLIP / SMPL seams
    def init_clip(self, visual_state_dict=None, encoded_text=None, encoded_face_text=None, encoded_back_text=None,
                  clip_model_path=None, bpe_path=None):
        """main.py:258-288.  Either pass the ViT-B/32 visual state dict and the encoded prompt [1,512] (+ face / back
        prompts when the conf enables them), or let init_clip encode the conf's prompts itself:

        * with ``clip_model_path`` given, or without the ``clip`` package: on the GPU from openai's ``ViT-B-32.pt``
          (``clip_model_path``, else ``$AVC_CLIP_MODEL``, else ``~/.cache/clip/ViT-B-32.pt`` where ``clip.load`` saves
          it) and the BPE merges ``bpe_simple_vocab_16e6.txt.gz`` (``bpe_path``, else next to the model file);
        * otherwise through the ``clip`` package, as the reference does."""
        from .clip_vit import ClipImageTower
        if visual_state_dict is None and (clip_model_path is not None or not _clip_importable()):
            visual_state_dict, encoded_text, encoded_face_text, encoded_back_text = \
                self._encode_prompts(clip_model_path, bpe_path)
        if visual_state_dict is None:
            import clip                                                   # noqa: F401 (optional dependency)
            model, _ = clip.load("ViT-B/32", jit=False)
            model = model.eval().requires_grad_(False).to(self.device)
            enc = lambda key: model.encode_text(clip.tokenize([self.conf.get_string(key)]).to(self.device)).detach().float()
            encoded_text = enc("clip.prompt")
            if self.use_face_prompt:
                encoded_face_text = enc("clip.face_prompt")
            if self.use_back_prompt:
                encoded_back_text = enc("clip.back_prompt")
            visual_state_dict = model.visual.state_dict()
        if self.use_face_prompt and encoded_face_text is None:
            raise ValueError("train.use_face_prompt is set: init_clip needs encoded_face_text (clip.face_prompt)")
        if self.use_back_prompt and encoded_back_text is None:
            raise ValueError("train.use_back_prompt is set: init_clip needs encoded_back_text (clip.back_prompt)")
        self.clip_tower = ClipImageTower(visual_state_dict, device=self.device)
        prep = lambda t: None if t is None else t.detach().float().reshape(1, -1).to(self.device)
        self.encoded_text, self.encoded_face_text, self.encoded_back_text = \
            prep(encoded_text), prep(encoded_face_text), prep(encoded_back_text)

    def _encode_prompts(self, clip_model_path=None, bpe_path=None):
        """The ``clip``-free half of init_clip: read ViT-B-32.pt, tokenize the prompt (+ face / back prompts) and encode
        them in one batch on the GPU.  Returns (visual state dict, prompt, face prompt, back prompt) with [1,512]
        embeddings (None for a prompt the conf does not use).  The text tower is dropped afterwards."""
        from .clip_text import ClipTextTower, load_clip_model
        from .clip_tokenizer import ClipTokenizer
        model_path = clip_model_path or os.environ.get("AVC_CLIP_MODEL") or \
            os.path.join(os.path.expanduser("~"), ".cache", "clip", "ViT-B-32.pt")
        if not os.path.isfile(model_path):
            raise FileNotFoundError(f"init_clip: the CLIP ViT-B/32 model file {model_path} does not exist (pass "
                                    "clip_model_path or set AVC_CLIP_MODEL to openai's ViT-B-32.pt)")
        bpe_path = bpe_path or os.path.join(os.path.dirname(model_path), "bpe_simple_vocab_16e6.txt.gz")
        if not os.path.isfile(bpe_path):
            raise FileNotFoundError(f"init_clip: the CLIP BPE merges file {bpe_path} does not exist (pass bpe_path; "
                                    "openai ships bpe_simple_vocab_16e6.txt.gz inside the clip package)")
        keys = ["clip.prompt"] + ["clip.face_prompt"] * self.use_face_prompt + ["clip.back_prompt"] * self.use_back_prompt
        prompts = [self.conf.get_string(k) for k in keys]
        for k, text in zip(keys, prompts):
            logging.info("%s: %s", k, text)
        visual, text_sd = load_clip_model(model_path)
        tower = ClipTextTower(text_sd, device=self.device)
        tokens = ClipTokenizer(bpe_path).tokenize(prompts, context_length=tower.context)
        emb = dict(zip(keys, tower.encode_text(tokens).split(1)))
        del tower, text_sd
        return visual, emb["clip.prompt"], emb.get("clip.face_prompt"), emb.get("clip.back_prompt")

    def init_smpl(self, v=None, f=None, smpl=None, v_shaped=None, pose=None):
        """main.py:290-335: the posed template ``self.v`` [1,V,3] / ``self.f`` [F,3] the silhouette rasteriser draws.
        Either pass ``v`` / ``f`` directly, or the SMPL tensors ``smpl`` = dict(J_regressor, parents, posedirs,
        lbs_weights, faces) with ``v_shaped`` [1,V,3] (``dataset.template_obj``, main.py:316) and ``pose`` [1,24,3]
        axis-angle (``stand_pose.npy`` / the T-pose of main.py:307-309): then ``my_lbs`` runs as in main.py:322-328."""
        if v is None:
            if smpl is None:
                raise ValueError("init_smpl: smplx / SMPL_NEUTRAL.pkl are not available here -- pass v, f or the SMPL tensors")
            from .lbs import my_lbs
            if v_shaped is None:
                from .views import read_obj
                v_shaped = torch.from_numpy(read_obj(self.conf.get_string("dataset.template_obj"))[0]).reshape(1, -1, 3)
            if pose is None:
                if self.pose_type != "t_pose":
                    raise ValueError("init_smpl: pass pose (ShapeGen/output/stand_pose.npy) for pose_type stand_pose")
                pose = np.zeros([1, 24, 3], dtype=np.float32)
                pose[:, 0, 0] = np.pi / 2
            pose = torch.as_tensor(pose, dtype=torch.float32).reshape(1, -1, 3).to(self.device)
            v, _ = my_lbs(torch.as_tensor(v_shaped, dtype=torch.float32).to(self.device), pose.reshape(1, -1), None, None,
                          smpl["posedirs"], smpl["J_regressor"], smpl["parents"], smpl["lbs_weights"], pose2rot=True)
            f = smpl["faces"]
        self.v = torch.as_tensor(v, dtype=torch.float32).reshape(1, -1, 3).to(self.device)
        self.f = np.asarray(f.cpu() if torch.is_tensor(f) else f).astype(np.int64)

    def set_process_group(self, pg):
        """View-sharded data parallelism (SURVEY.md 8e): rank r of N takes draw number step * N + r of the ONE seeded
        stream (``StepSampler.draw_for_rank``), the flat gradient is all-reduced once per step inside the trainer."""
        import torch.distributed as dist
        self.process_group = pg
        self.rank, self.world = (dist.get_rank(pg), dist.get_world_size(pg)) if pg is not None else (0, 1)
        if self.trainer is not None:
            self.trainer.pg, self.trainer.world = pg, self.world

    def _ensure_trainer(self):
        from .trainer import AppearanceTrainer
        if self.trainer is None:
            if self.clip_tower is None:
                raise RuntimeError("call init_clip() first (main.py:970-972)")
            self.trainer = AppearanceTrainer(self.renderer, self.clip_tower, self.encoded_text, lr=self.learning_rate,
                                             igr_weight=self.igr_weight, mask_weight=self.mask_weight,
                                             clip_weight=1.0 if self.clip_weight is None else self.clip_weight,
                                             process_group=self.process_group, device=self.device,
                                             texture_cast_light=self.texture_cast_light,
                                             add_no_texture=self.add_no_texture)
            self.trainer.iter_step = self.iter_step
            if self._pending_optimizer_state is not None:      # checkpoint loaded before init_clip() (the CLI order)
                self._load_optimizer_state_dict(self._pending_optimizer_state)
                self._pending_optimizer_state = None
        return self.trainer

    # ------------------------------------------------------------------ train_clip (main.py:337-566)
    def train_clip(self, max_steps: Optional[int] = None, view_source=None, log=print, validate: bool = True):
        """The appearance-optimisation loop.  ``view_source(step) -> view`` overrides the per-step view (tests /
        synthetic workloads); by default every step draws a camera, rasterises the template (``init_smpl``) and prepares
        the silhouette rays on the device, one step ahead of the optimiser."""
        if not (self.use_silhouettes and self.extra_color):
            raise NotImplementedError("avatarclip_b200 implements the train_clip configurations of the shipped confs: "
                                      "use_silhouettes and extra_color on (all 179 train_clip confs); add_no_texture / "
                                      "texture_cast_light / use_bg_aug / face and back prompts as the conf says (DESIGN.md)")
        from .views import ViewBuilder
        tr = self._ensure_trainer()
        self.writer = self._make_writer()
        sampler = builder = None
        if view_source is None:
            if self.v is None:
                raise RuntimeError("call init_smpl() first (main.py:973): train_clip rasterises the posed template")
            sampler = StepSampler(self.seed, self.use_face_prompt, self.head_height, self.use_bg_aug,
                                  rng=np.random if self.seed is not None else None,
                                  cast_light=self.add_no_texture or self.texture_cast_light)            # main.py:425
            builder = ViewBuilder(self.v, self.f, self.max_ray_num, self.mask_weight, self.device,
                                  image_size=self.dataset.H,
                                  camera_angle_x=2 * np.arctan(0.5 * self.dataset.W / self.dataset.focal))
        res_step = self.end_iter - self.iter_step
        texts = {"body": self.encoded_text, "face": self.encoded_face_text, "back": self.encoded_back_text}
        draw = lambda i: sampler.draw_for_rank(i, self.rank, self.world)
        pending = builder.submit(draw(0)) if builder is not None else None
        for iter_i in range(res_step):
            if iter_i == 30010 or (max_steps is not None and iter_i >= max_steps):      # main.py:346-347
                break
            if builder is not None:
                view = builder.finish(pending)
                nxt = iter_i + 1
                pending = builder.submit(draw(nxt)) if nxt < res_step else None             # lookahead: overlaps this step
                which = view.draw.prompt
                if which == "back" and not self.use_back_prompt:
                    which = "body"
                tr.set_text(texts[which])                                                 # main.py:499-507
            else:
                view = view_source(self.iter_step)
                if not torch.is_tensor(view.rays_o) or not view.rays_o.is_cuda:
                    from .trainer import DeviceView
                    view = DeviceView(view, self.device)
            loss = tr.step(view, lr=self.current_lr(), cos_anneal=self.get_cos_anneal_ratio())
            self.iter_step += 1
            if not isinstance(self.writer, _NullWriter):
                sc = tr.scalars                                                           # main.py:542-547 (one read-back)
                vals = torch.stack([loss.reshape(()), sc[0], sc[1], tr.cos[0], tr._out["s_val"].mean(), sc[3]]).tolist()
                for name, v in zip(("Loss/loss", "Loss/color_loss", "Loss/eikonal_loss", "Loss/cosine", "Statistics/s_val",
                                    "Statistics/psnr"), vals):
                    self.writer.add_scalar(name, v, self.iter_step)
            if self.iter_step % self.report_freq == 0:
                log(self.base_exp_dir)
                log("iter:{:8>d} loss = {} lr={}".format(self.iter_step, float(loss), self.current_lr()))
            if self.iter_step % self.save_freq == 0:
                self.save_checkpoint()
            if validate and self.iter_step % self.val_freq == 0 and self.dataset is not None and self.dataset.n_images > 58:
                self.validate_image(idx=58)                                               # main.py:556-557
            if validate and self.iter_step % self.val_mesh_freq == 0:
                self.validate_mesh()
        return self.iter_step

    # ------------------------------------------------------------------ train (main.py:180-256)
    def _ensure_optimizer(self):
        if self.optimizer is None:
            fp = self.renderer.flat_params(self.device)
            self.optimizer = torch.optim.Adam(self._all_params(), lr=self.learning_rate)        # main.py:141-145
            assert fp.is_homed()
            if self._pending_optimizer_state is not None:
                self.optimizer.load_state_dict(self._pending_optimizer_state)
                self._pending_optimizer_state = None
        return self.optimizer

    def train(self, max_steps: Optional[int] = None, log=print, validate: bool = True):
        """NeuS pre-fit on the rendered template views (main.py:180-256): the reference's loop over the differentiable
        ``NeuSRenderer.render`` seam (``loss.backward()`` + ``torch.optim.Adam``, unmodified protocol)."""
        import torch.nn.functional as F
        if self.dataset is None or self.dataset.n_images == 0:
            raise RuntimeError("--mode train needs dataset.data_dir with transforms_train.json + img/*.png")
        opt = self._ensure_optimizer()
        self.writer = self._make_writer()
        self.update_learning_rate()
        res_step = self.end_iter - self.iter_step
        image_perm = self.get_image_perm()
        for iter_i in range(res_step):
            if max_steps is not None and iter_i >= max_steps:
                break
            data = self.dataset.gen_random_rays_at(image_perm[self.iter_step % len(image_perm)], self.batch_size)
            rays_o, rays_d, true_rgb, mask = data[:, :3], data[:, 3:6], data[:, 6:9], data[:, 9:10]
            near, far = self.dataset.near_far_from_sphere(rays_o, rays_d)
            background_rgb = torch.ones([1, 3], device=self.device) if self.use_white_bkgd else None
            mask = (mask > 0.5).float() if self.mask_weight > 0.0 else torch.ones_like(mask)
            mask_sum = mask.sum() + 1e-5
            out = self.renderer.render(rays_o, rays_d, near, far, background_rgb=background_rgb,
                                       cos_anneal_ratio=self.get_cos_anneal_ratio())
            color_fine, weight_sum = out["color_fine"], out["weight_sum"]
            color_error = (color_fine - true_rgb) * mask
            color_fine_loss = F.l1_loss(color_error, torch.zeros_like(color_error), reduction="sum") / mask_sum
            psnr = 20.0 * torch.log10(1.0 / (((color_fine - true_rgb) ** 2 * mask).sum() / (mask_sum * 3.0)).sqrt())
            eikonal_loss = out["gradient_error"]
            mask_loss = F.binary_cross_entropy(weight_sum.clip(1e-3, 1.0 - 1e-3), mask)
            loss = color_fine_loss + eikonal_loss * self.igr_weight + mask_loss * self.mask_weight
            opt.zero_grad()
            loss.backward()
            opt.step()
            self.iter_step += 1
            w = self.writer
            w.add_scalar("Loss/loss", loss, self.iter_step)
            w.add_scalar("Loss/color_loss", color_fine_loss, self.iter_step)
            w.add_scalar("Loss/eikonal_loss", eikonal_loss, self.iter_step)
            w.add_scalar("Statistics/s_val", out["s_val"].mean(), self.iter_step)
            w.add_scalar("Statistics/cdf", (out["cdf_fine"][:, :1] * mask).sum() / mask_sum, self.iter_step)
            w.add_scalar("Statistics/weight_max", (out["weight_max"] * mask).sum() / mask_sum, self.iter_step)
            w.add_scalar("Statistics/psnr", psnr, self.iter_step)
            if self.iter_step % self.report_freq == 0:
                log(self.base_exp_dir)
                log("iter:{:8>d} loss = {} lr={}".format(self.iter_step, float(loss), opt.param_groups[0]["lr"]))
            if self.iter_step % self.save_freq == 0:
                self.save_checkpoint()
            if validate and self.iter_step % self.val_freq == 0:
                self.validate_image()
            if validate and self.iter_step % self.val_mesh_freq == 0:
                self.validate_mesh()
            self.update_learning_rate()
            if self.iter_step % len(image_perm) == 0:
                image_perm = self.get_image_perm()
        return self.iter_step

    # ------------------------------------------------------------------ checkpoints (main.py:601-632)
    def _all_params(self):
        return list(self.sdf_network.parameters()) + list(self.deviation_network.parameters()) + \
            list(self.color_network.parameters())

    def _optimizer_state_dict(self):
        """torch.optim.Adam-format state dict (parameter order of main.py:141-143: sdf, variance, colour) -- from the
        torch optimizer of ``train`` or built from the fused Adam's flat moment vectors of ``train_clip``, so the
        reference can resume from either."""
        if self.optimizer is not None and self.trainer is None:
            return self.optimizer.state_dict()
        params = self._all_params()
        state = {}
        tr = self.trainer
        if tr is not None and tr.iter_step > 0:
            slot = {id(p): (o, m) for p, o, m in tr.fp.slots}
            for i, p in enumerate(params):
                o, m = slot[id(p)]
                state[i] = {"step": torch.tensor(float(tr.iter_step)),
                            "exp_avg": tr.exp_avg[o:o + m].view(p.shape).clone(),
                            "exp_avg_sq": tr.exp_avg_sq[o:o + m].view(p.shape).clone()}
        group = {"lr": self.current_lr(), "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0, "amsgrad": False,
                 "maximize": False, "foreach": None, "capturable": False, "differentiable": False, "fused": None,
                 "params": list(range(len(params)))}
        return {"state": state, "param_groups": [group]}

    def _load_optimizer_state_dict(self, sd):
        """optimizer.load_state_dict of main.py:606 for the fused Adam: per-parameter moments -> the flat moment vectors.
        When the trainer does not exist yet (``Runner(..., is_continue=True)`` runs before ``init_clip``, main.py:963-972)
        the state is kept and applied as soon as the trainer (or ``train``'s torch optimizer) is built."""
        if not sd or not sd.get("state"):
            return
        if self.trainer is None:
            self._pending_optimizer_state = sd
            if self.clip_tower is not None:
                self._ensure_trainer()                 # builds the trainer and applies the pending state
            return
        tr = self.trainer
        params = self._all_params()
        slot = {id(p): (o, m) for p, o, m in tr.fp.slots}
        for i, p in enumerate(params):
            st = sd["state"].get(i)
            if st is None:
                continue
            o, m = slot[id(p)]
            tr.exp_avg[o:o + m].copy_(st["exp_avg"].reshape(-1).to(self.device))
            tr.exp_avg_sq[o:o + m].copy_(st["exp_avg_sq"].reshape(-1).to(self.device))

    def save_checkpoint(self):
        checkpoint = {
            "sdf_network_fine": self.sdf_network.state_dict(),
            "variance_network_fine": self.deviation_network.state_dict(),
            "color_network_fine": self.color_network.state_dict(),
            "optimizer": self._optimizer_state_dict(),
            "iter_step": self.iter_step,
        }
        os.makedirs(os.path.join(self.base_exp_dir, "checkpoints"), exist_ok=True)
        path = os.path.join(self.base_exp_dir, "checkpoints", "ckpt_{:0>6d}.pth".format(self.iter_step))
        torch.save(checkpoint, path)
        return path

    def load_checkpoint(self, checkpoint_name):
        path = checkpoint_name if os.path.isabs(checkpoint_name) else \
            os.path.join(self.base_exp_dir, "checkpoints", checkpoint_name)
        ck = torch.load(path, map_location=self.device, weights_only=False)
        self.sdf_network.load_state_dict(ck["sdf_network_fine"])
        self.deviation_network.load_state_dict(ck["variance_network_fine"])
        self.color_network.load_state_dict(ck["color_network_fine"])
        self.iter_step = ck["iter_step"]
        if self.trainer is not None:
            self.trainer.iter_step = self.iter_step
        if self.optimizer is not None and self.trainer is None:
            self.optimizer.load_state_dict(ck["optimizer"])
        else:
            self._load_optimizer_state_dict(ck.get("optimizer", {}))

    def load_pretrain(self, checkpoint_name):
        ck = torch.load(checkpoint_name, map_location=self.device, weights_only=False)
        self.sdf_network.load_state_dict(ck["sdf_network_fine"])
        self.deviation_network.load_state_dict(ck["variance_network_fine"])
        self.color_network.load_state_dict(ck["color_network_fine"], strict=False)      # no extra_lin in the file

    # ------------------------------------------------------------------ validation (main.py:634-919)
    def _render_batches(self, rays_o, rays_d, background_rgb=None, keys=("color_fine",)):
        """Chunked no-grad render of [N,3] rays in ``batch_size`` pieces like main.py:751-769 -> dict of [N, ...]."""
        outs = {k: [] for k in keys}
        with torch.no_grad():
            for ro, rd in zip(rays_o.split(self.batch_size), rays_d.split(self.batch_size)):
                near, far = self.dataset.near_far_from_sphere(ro, rd)
                out = self.renderer.render(ro, rd, near, far, cos_anneal_ratio=self.get_cos_anneal_ratio(),
                                           background_rgb=background_rgb)
                for k in keys:
                    outs[k].append(out[k])
        return {k: torch.cat(v, 0) for k, v in outs.items()}

    def render_image(self, pose, resolution_level=1):
        """Full-image render of ``extra_color_fine`` (``color_fine`` for a network without the extra head) for a
        camera-to-world pose -> [H, W, 3] tensor."""
        ro, rd = self.dataset.gen_rays_pose(pose, resolution_level)
        H, W = ro.shape[:2]
        ckey = "extra_color_fine" if self.extra_color else "color_fine"
        o = self._render_batches(ro.reshape(-1, 3), rd.reshape(-1, 3), keys=(ckey,))
        return o[ckey].reshape(H, W, 3)

    def validate_image(self, idx=-1, resolution_level=-1):
        """main.py:741-820: colour, extra colour and normal images of training camera ``idx``."""
        import cv2 as cv
        if idx < 0:
            idx = np.random.randint(self.dataset.n_images)
        print("Validate: iter: {}, camera: {}".format(self.iter_step, idx))
        if resolution_level < 0:
            resolution_level = self.validate_resolution_level
        ro, rd = self.dataset.gen_rays_at(idx, resolution_level=resolution_level)
        H, W, _ = ro.shape
        bg = torch.ones([1, 3], device=self.device) if self.use_white_bkgd else None
        o = self._render_batches(ro.reshape(-1, 3), rd.reshape(-1, 3), bg,
                                 keys=("color_fine",) + (("extra_color_fine",) if self.extra_color else ())
                                 + ("gradients", "weights", "inside_sphere"))
        img_fine = (o["color_fine"].cpu().numpy().reshape([H, W, 3, -1]) * 255).clip(0, 255)
        extra_img = (o["extra_color_fine"].cpu().numpy().reshape([H, W, 3, -1]) * 255).clip(0, 255) if self.extra_color else None
        normals = (o["gradients"] * o["weights"][:, :, None] * o["inside_sphere"][..., None]).sum(dim=1).cpu().numpy()
        rot = np.linalg.inv(self.dataset.poses[idx, :3, :3].detach().cpu().numpy())
        normal_img = (np.matmul(rot[None, :, :], normals[:, :, None]).reshape([H, W, 3, -1]) * 128 + 128).clip(0, 255)
        for d in ("validations_fine", "validations_extra_fine", "normals"):
            os.makedirs(os.path.join(self.base_exp_dir, d), exist_ok=True)
        name = "{:0>8d}_{}_{}.png".format(self.iter_step, 0, idx)
        cv.imwrite(os.path.join(self.base_exp_dir, "validations_fine", name),
                   np.concatenate([img_fine[..., 0], self.dataset.image_at(idx, resolution_level=resolution_level)]))
        if extra_img is not None:
            cv.imwrite(os.path.join(self.base_exp_dir, "validations_extra_fine", name),
                       cv.cvtColor(extra_img[..., 0].astype(np.float32), cv.COLOR_RGB2BGR))
        cv.imwrite(os.path.join(self.base_exp_dir, "normals", name), normal_img[..., 0])
        return img_fine[..., 0], None if extra_img is None else extra_img[..., 0], normal_img[..., 0]

    def validate_mesh(self, world_space=False, resolution=256, threshold=0.0):
        """main.py:850-919: iso-surface of the SDF + per-vertex colour from the best of six axis views -> PLY."""
        from .handoff import write_ply
        bmin = self.dataset.object_bbox_min if self.dataset is not None else np.array([-1.01, -1.01, -1.01])
        bmax = self.dataset.object_bbox_max if self.dataset is not None else np.array([1.01, 1.01, 1.01])
        bound_min, bound_max = torch.tensor(bmin, dtype=torch.float32), torch.tensor(bmax, dtype=torch.float32)
        vertices, triangles = self.renderer.extract_geometry(bound_min, bound_max, resolution=resolution, threshold=threshold)
        os.makedirs(os.path.join(self.base_exp_dir, "meshes"), exist_ok=True)
        path = os.path.join(self.base_exp_dir, "meshes", "{:0>8d}.ply".format(self.iter_step))
        if vertices.shape[0] == 0:
            write_ply(path, vertices, triangles, np.zeros((0, 3), dtype=np.uint8))
            return path
        pt = torch.from_numpy(vertices).to(self.device).float()
        bg = torch.ones([1, 3], device=self.device) if self.use_white_bkgd else None
        ckey = "extra_color_fine" if self.extra_color else "color_fine"
        rgb_final = diff_final = None
        for eye in ([0, 0, 2], [0, 0, -2], [0, 2, 0], [0, -2, 0], [2, 0, 0], [-2, 0, 0]):                  # main.py:861-868
            ro = torch.tensor(eye, dtype=torch.float32, device=self.device).reshape(1, 3).repeat(pt.shape[0], 1)
            rd = pt - ro
            dist = torch.norm(rd, dim=-1)
            rd = rd / dist.reshape(-1, 1)
            o = self._render_batches(ro, rd, bg, keys=(ckey, "weights", "mid_z_vals"))
            rgb = o[ckey]
            depth = (o["mid_z_vals"] * o["weights"]).sum(dim=1)
            diff = (depth - dist).abs()
            if rgb_final is None:
                rgb_final, diff_final = rgb.clone(), diff.clone()
            else:
                ind = diff_final > diff                                                                     # main.py:907-911
                rgb_final[ind] = rgb[ind]
                diff_final[ind] = diff[ind]
        write_ply(path, vertices, triangles, to8b(rgb_final.cpu().numpy()))
        logging.info("End")
        return path

    def render_geometry_cast_light(self):
        """main.py:634-739: 512 x 512 close-up of the head, texture x Lambert shading (ambience 0, black background)."""
        import cv2 as cv
        if not self.extra_color:
            raise RuntimeError("render_geometry_cast_light shades the extra colour (main.py:705-723): the conf has "
                               "model.rendering_network.extra_color = False")
        eye = sphere_coord(0.0, 0.0, 0.5)
        at = np.array([0, self.head_height, 0.3])
        eye = eye + at
        pose = lookat(eye, at, np.array([0, 1, 0]))
        ro, rd = self.dataset.gen_rays_pose(pose, 0.5)
        H, W = ro.shape[0], ro.shape[1]
        light = sphere_coord(0 + np.random.uniform(-np.pi / 4, np.pi / 4), 0 + np.random.uniform(-np.pi / 4, np.pi / 4))
        np.random.choice(np.arange(10, 20))                                                 # main.py:669 (stream position)
        light = torch.from_numpy(light).float().to(self.device)
        o = self._render_batches(ro.reshape(-1, 3), rd.reshape(-1, 3), None,
                                 keys=("extra_color_fine", "gradients", "weights", "weight_sum"))
        normals = (o["gradients"] * o["weights"][:, :, None]).sum(dim=1)
        normals = normals / (torch.norm(normals, dim=-1, keepdim=True) + 1e-7)
        ld = light / (torch.norm(light) + 1e-7)
        shading = (normals * ld[None]).sum(-1, keepdim=True).clamp(min=0, max=1)
        shading[torch.isnan(shading)] = 1.0
        wsum = o["weight_sum"].reshape(-1)
        shading[wsum < 0.5] = 1.0
        img = (o["extra_color_fine"] * shading).clamp(min=0, max=1).cpu().numpy().reshape(H, W, 3)
        path = os.path.join(self.base_exp_dir, "cast_light_texture_head_black.png")
        cv.imwrite(path, cv.cvtColor(to8b(img), cv.COLOR_RGB2BGR))
        return path


def main(argv=None):
    logging.basicConfig(level=logging.INFO, format="[%(filename)s:%(lineno)s - %(funcName)20s() ] %(message)s")
    p = argparse.ArgumentParser()                                   # main.py:953-961
    p.add_argument("--conf", type=str, default="./confs/base.conf")
    p.add_argument("--mode", type=str, default="train")
    p.add_argument("--mcube_threshold", type=float, default=0.0)
    p.add_argument("--is_continue", default=False, action="store_true")
    p.add_argument("--gpu", type=int, default=0)
    p.add_argument("--case", type=str, default="smpl")
    args = p.parse_args(argv)
    torch.cuda.set_device(args.gpu)
    if args.mode in ("validate_mesh", "render_geometry_cast_light"):      # main.py:965-967: inference on the last checkpoint
        args.is_continue = True
    runner = Runner(args.conf, args.mode, args.case, args.is_continue, device=f"cuda:{args.gpu}")
    if args.mode == "train":                                        # main.py:970-979
        runner.train()
    elif args.mode == "validate_mesh":
        runner.validate_mesh(world_space=True, resolution=512, threshold=args.mcube_threshold)   # world_space is unused (:850)
        runner.render_geometry_cast_light()
    elif args.mode == "train_clip":
        runner.init_clip()
        runner.init_smpl()
        runner.train_clip()
    elif args.mode == "render_geometry_cast_light":
        runner.render_geometry_cast_light()
    else:
        raise SystemExit(f"unknown mode {args.mode!r}")


if __name__ == "__main__":
    main()
