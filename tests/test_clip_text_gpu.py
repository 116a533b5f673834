"""GPU checks of the CLIP text tower (avc_clip_encode_text) against the CPU oracle (oracle/clip_text.py: the published
architecture restated and cross-checked against HF transformers; parity unpinned w.r.t. openai/CLIP itself).

One prompt (M = 77 token rows) runs every GEMM on the wgmma kernel, three prompts (M = 231) on the mma.sync kernel."""
import ctypes as C
import functools
import sys

import pytest
import torch

import util_neus as U
from oracle import clip_text as ot
from oracle import clip_vit as ov
from oracle.pin_clip_text import sample_tokens

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _text_state(seed=0, layers=12):
    return ot.random_text_state(ot.TextConf(layers=layers), seed=seed)


def _tower(seed=0, layers=12):
    from avatarclip_b200.clip_text import ClipTextTower
    return ClipTextTower(_text_state(seed, layers), device="cuda")


@pytest.mark.parametrize("eot_positions", [[76], [3, 40, 76]], ids=["1", "3"])
def test_encode_text_matches_oracle(eot_positions):
    """Full-size random weights; end-of-text at positions 3, 40 and 76 (76: the whole context is text)."""
    tower = _tower()
    tok = sample_tokens(ot.TextConf(), eot_positions, seed=len(eot_positions))
    want = ot.encode_text(_text_state(), tok)
    got = tower.encode_text(tok.cuda())
    torch.cuda.synchronize()
    err = U.rel_to_max(got, want)
    # one encode, timed with CUDA events after a warm-up call
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    tok_d = tok.cuda()
    start.record()
    for _ in range(10):
        tower.encode_text(tok_d)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / 10
    U.log_parity("clip_text_tower", {"prompts": len(eot_positions), "emb_rel_to_max": err, "ms_per_encode": ms})
    print(f"prompts={len(eot_positions)}: embedding rel-to-max err {err:.2e}, {ms:.3f} ms per encode")
    assert got.shape == (len(eot_positions), 512)
    assert err < 5e-3       # fp16 GEMM operands (as in the reference's CUDA path), fp32 accumulate


def test_clip_loss_with_the_product_text_embedding():
    """The CLIP loss 1 - cos of main.py:513 with both embeddings from the product against both from the oracle."""
    from avatarclip_b200.clip_vit import ClipImageTower
    sd_v = ov.random_vit_state(seed=1)
    image = ClipImageTower(sd_v, device="cuda")
    text = _tower()
    tok = sample_tokens(ot.TextConf(), [12], seed=5)
    g = torch.Generator().manual_seed(2)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, 224), torch.linspace(0, 1, 224), indexing="ij")
    canvas = (torch.stack([0.5 + 0.4 * torch.sin(6 * xx + 2 * yy), 0.5 + 0.4 * torch.cos(5 * yy), xx * yy], -1)
              + 0.1 * torch.randn(224, 224, 3, generator=g)).clamp(0, 1)
    cos_o = ov.clip_cosine(sd_v, canvas, ot.encode_text(_text_state(), tok))
    cos_p = image.cosine(canvas[None].cuda(), text.encode_text(tok.cuda())).cpu()[0]
    rel = abs((1 - cos_o.item()) - (1 - cos_p.item())) / abs(1 - cos_o.item())
    print(f"cos oracle {cos_o.item():.6f} product {cos_p.item():.6f}: loss rel err {rel:.2e}")
    assert rel < 1e-3


def test_runner_init_clip_from_the_model_file_without_the_clip_package(tmp_path, monkeypatch):
    """init_clip(clip_model_path, bpe_path) with `import clip` failing: the conf's three prompts are tokenized and encoded
    in one batch from a torch.save'd openai state dict; then the training loop runs on those embeddings."""
    from avatarclip_b200.clip_text import ClipTextTower, load_clip_model
    from avatarclip_b200.clip_tokenizer import ClipTokenizer
    from avatarclip_b200.workload import random_vit_state, synthetic_body_mesh
    from test_clip_text_cpu import synthetic_bpe
    from test_runner import _runner
    monkeypatch.setitem(sys.modules, "clip", None)
    _, gz, _, _ = synthetic_bpe(tmp_path)
    sd = {"visual." + k: v for k, v in random_vit_state(seed=0, layers=2).items()}
    sd.update(_text_state(seed=4, layers=2))
    sd["logit_scale"] = torch.tensor(4.6052)
    model = str(tmp_path / "ViT-B-32.pt")
    torch.save(sd, model)
    r = _runner(tmp_path, "cuda")
    assert r.use_face_prompt and r.use_back_prompt
    r.init_clip(clip_model_path=model, bpe_path=gz)
    prompts = [r.conf.get_string(k) for k in ("clip.prompt", "clip.face_prompt", "clip.back_prompt")]
    want = ClipTextTower(load_clip_model(model)[1], device="cuda").encode_text(ClipTokenizer(gz).tokenize(prompts))
    got = torch.cat([r.encoded_text, r.encoded_face_text, r.encoded_back_text])
    assert r.encoded_text.shape == (1, 512)
    # the same kernels on the same batch: only the order of the split-K fp32 atomics varies between two encodes, which
    # can flip the fp16 rounding of a GEMM operand (measured 1.1e-4; the image tower's run-to-run spread is up to 1e-3),
    # while two different prompts differ by O(1)
    assert U.rel_to_max(got, want) < 1e-3
    assert r.clip_tower.cfg.layers == 2
    v, f = synthetic_body_mesh(12, 16)
    r.init_smpl(v, f)
    assert r.train_clip(max_steps=2, log=lambda m: None, validate=False) == 2


def test_unsupported_shapes_and_token_ids_are_rejected():
    from avatarclip_b200 import _lib
    from avatarclip_b200.clip_text import ClipTextCfg, _bind
    L = _lib.lib()
    _bind(L)
    size = C.c_size_t()
    ok = dict(context=77, vocab=49408, width=512, layers=12, heads=8, mlp=2048, out_dim=512)
    assert L.avc_clip_text_workspace_bytes(C.byref(ClipTextCfg(**ok)), 3, C.byref(size)) == 0 and size.value > 0
    for bad in (dict(heads=4), dict(context=129), dict(mlp=2000), dict(layers=25), dict(width=1088, heads=17)):
        assert L.avc_clip_text_workspace_bytes(C.byref(ClipTextCfg(**{**ok, **bad})), 1, C.byref(size)) == -1, bad
    tower = _tower(layers=2)
    tok = sample_tokens(ot.TextConf(), [5])
    for bad_id in (49408, -1):
        t = tok.clone()
        t[0, 2] = bad_id
        with pytest.raises(_lib.AvcError, match="token ids"):
            tower.encode_text(t.cuda())


@pytest.mark.parametrize("context", [1, 2, 128])
def test_encode_text_context_lengths(context):
    """Contexts of 1 and 128 tokens (the causal attention's limit) on a two-layer tower."""
    from avatarclip_b200.clip_text import ClipTextTower
    conf = ot.TextConf(context=context, vocab=1000, layers=2)
    sd = ot.random_text_state(conf, seed=context)
    g = torch.Generator().manual_seed(context)
    tok = torch.randint(1, 999, (3, context), generator=g, dtype=torch.int32)
    tok[0, -1] = 999
    tok[1, context // 2] = 999
    want = ot.encode_text(sd, tok, conf)
    got = ClipTextTower(sd, device="cuda").encode_text(tok.cuda()).cpu()
    err = U.rel_to_max(got, want)
    U.log_parity("clip_text_context", {"context": context, "emb_rel_to_max": err})
    assert err < 1.7e-3         # measured <= 4.39e-4 on an H100 (400 W)
