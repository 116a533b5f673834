"""CPU checks of the CLIP text path (avatarclip_b200/clip_tokenizer.py, clip_text.py, oracle/clip_text.py):

* the restated text tower against HF transformers ``CLIPTextModelWithProjection`` (oracle/pin_clip_text.py);
* the tokenizer against HF ``CLIPTokenizer`` on a synthetic BPE learned from the shipped confs' prompts (openai's
  ``bpe_simple_vocab_16e6.txt.gz`` is not on disk), written in both file formats;
* cleaning, the context-length error and truncation;
* ``load_clip_model`` on a TorchScript archive and on a plain state dict, with openai's key names;
* the ctypes mirrors of ``avc_clip_text_cfg`` / ``avc_clip_text_weights`` against the C layout."""
import ctypes as C
import glob
import gzip
import json
import os
import shutil
import subprocess
from collections import Counter

import pytest
import torch

import util_neus as U
from avatarclip_b200 import clip_tokenizer as CT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROMPT_KEYS = ("clip.prompt", "clip.face_prompt", "clip.back_prompt")
EDGE_STRINGS = [
    "hello   world\t\n  again ",                                   # repeated whitespace
    "it's the dog't they're we've I'm you'll he'd IT'S",           # the contraction alternatives
    "12345 0.5 2024x 3d",                                           # digit runs
    "!!!??...,;:-- (a) [b] {c} \"q\"",                             # punctuation runs
    "café naïve Straße Ünïcödé 東京 ok",                            # non-ASCII letters
]


def shipped_prompts(tmp_path):
    from avatarclip_b200 import conf as hocon
    root = U.reference_tree(tmp_path / "ref")
    confs = sorted(glob.glob(os.path.join(root, "confs", "**", "*.conf"), recursive=True))
    assert len(confs) == 180
    prompts = []
    for path in confs:
        c = hocon.parse_string(open(path).read())
        prompts += [c.get_string(k) for k in PROMPT_KEYS if c.get_string(k, default=None)]
    return prompts


def _merge(word, pair):
    out, i = [], 0
    while i < len(word):
        if i + 1 < len(word) and (word[i], word[i + 1]) == pair:
            out.append(word[i] + word[i + 1])
            i += 2
        else:
            out.append(word[i])
            i += 1
    return tuple(out)


def learn_merges(texts, n):
    """Byte-level BPE training on ``texts``: ``n`` times merge the most frequent adjacent pair (ties by the pair)."""
    table = CT.bytes_to_unicode()
    words = Counter()
    for t in texts:
        for piece in CT._PATTERN.findall(CT.clean(t)):
            s = "".join(table[b] for b in piece.encode("utf-8"))
            words[tuple(s[:-1]) + (s[-1] + "</w>",)] += 1
    merges = []
    for _ in range(n):
        pairs = Counter()
        for w, c in words.items():
            for p in zip(w, w[1:]):
                pairs[p] += c
        if not pairs:
            break
        best = max(pairs, key=lambda p: (pairs[p], p))
        merges.append(best)
        merged = Counter()
        for w, c in words.items():
            merged[_merge(w, best)] += c
        words = merged
    return merges


def synthetic_bpe(tmp_path, n_merges=300):
    """Merges learned from the shipped prompts, written as openai's ``.txt.gz`` and as HF ``vocab.json`` +
    ``merges.txt`` (vocabulary in openai's order).  Returns (prompts, gz path, vocab.json path, merges.txt path)."""
    prompts = shipped_prompts(tmp_path)
    merges = learn_merges(prompts, n_merges)
    lines = ["#version: 0.2"] + [f"{a} {b}" for a, b in merges]
    d = tmp_path / "bpe"
    d.mkdir(exist_ok=True)
    gz = d / "bpe_simple_vocab_16e6.txt.gz"
    with gzip.open(gz, "wt", encoding="utf-8") as f:
        f.write("\n".join(lines))
    tok = CT.ClipTokenizer(str(gz))
    (d / "vocab.json").write_text(json.dumps({s: i for s, i in sorted(tok.encoder.items(), key=lambda kv: kv[1])}))
    (d / "merges.txt").write_text("\n".join(lines) + "\n")
    return prompts, str(gz), str(d / "vocab.json"), str(d / "merges.txt")


def test_restated_text_tower_matches_transformers():
    from oracle import pin_clip_text
    assert pin_clip_text.main() < 1e-4


def test_tokenizer_matches_transformers_on_a_synthetic_bpe(tmp_path):
    from transformers import CLIPTokenizer
    prompts, gz, vocab_json, merges_txt = synthetic_bpe(tmp_path)
    assert len(prompts) > 500 and all(p.isascii() for p in prompts)     # ftfy would change none of them
    tok = CT.ClipTokenizer(gz)
    n = 256 + 256 + len(tok.merges)
    assert len(tok.merges) >= 200 and (tok.sot, tok.eot) == (n, n + 1)
    assert list(tok.encoder)[:2] == ["!", '"'] and tok.encoder["!</w>"] == 256
    assert tok.encoder["a</w>"] == 320 and tok.encoder["Ā"] == 188     # openai's "a</w>"; byte 0 after the 188 printable
    hf = CLIPTokenizer(vocab_json, merges_txt)
    assert (hf.bos_token_id, hf.eos_token_id) == (tok.sot, tok.eot)
    for text in prompts + EDGE_STRINGS:
        want = hf(text)["input_ids"]
        assert [tok.sot] + tok.encode(text) + [tok.eot] == want, text
    rows = tok.tokenize(prompts)
    assert rows.dtype == torch.int32 and rows.shape == (len(prompts), 77)
    assert (rows.argmax(dim=1) == torch.tensor([len(tok.encode(p)) + 1 for p in prompts])).all()
    assert int(rows.max()) == tok.eot and (rows[:, 0] == tok.sot).all()


def test_cleaning_context_length_and_truncation(tmp_path):
    assert CT.clean("  A&amp;amp;B \n\t  Two&lt;3　x ") == "a&b two<3 x"
    assert CT.clean("&amp;amp;") == "&"
    _, gz, _, _ = synthetic_bpe(tmp_path)
    tok = CT.ClipTokenizer(gz)
    assert tok.encode("A  Photo\n\nOF") == tok.encode("a photo of")
    long_text = " ".join(f"w{i}" for i in range(60))           # 120 tokens: "w" and each digit are pieces of their own
    with pytest.raises(RuntimeError, match="too long for context length 77"):
        tok.tokenize(long_text)
    row = tok.tokenize([long_text, "a"], truncate=True)
    full = [tok.sot] + tok.encode(long_text)
    assert row[0, :76].tolist() == full[:76] and int(row[0, 76]) == tok.eot
    assert int(row[0].argmax()) == 76
    assert row[1, :3].tolist() == [tok.sot] + tok.encode("a") + [tok.eot] and int(row[1, 3:].abs().sum()) == 0


def small_openai_state(text_layers=2, vision_layers=1, seed=0):
    """A full openai/CLIP state dict (``visual.*`` + text tower + ``logit_scale``) at small widths."""
    from oracle import clip_text as ot
    from oracle import clip_vit as ov
    vconf = ov.ViTConf(image_size=64, patch=32, width=128, layers=vision_layers, heads=2, mlp=256, out_dim=64)
    tconf = ot.TextConf(context=77, vocab=1000, width=128, layers=text_layers, heads=2, mlp=256, out_dim=64)
    sd = {"visual." + k: v for k, v in ov.random_vit_state(vconf, seed=seed).items()}
    sd.update(ot.random_text_state(tconf, seed=seed + 1))
    sd["logit_scale"] = torch.tensor(4.6052)
    return sd


def _module_tree(sd):
    """A TorchScript-able module whose state_dict() is ``sd`` (keys become nested submodules and buffers)."""
    class Node(torch.nn.Module):
        def forward(self, x: torch.Tensor) -> torch.Tensor:
            return x

    root = Node()
    for key, value in sd.items():
        *path, leaf = key.split(".")
        m = root
        for name in path:
            if not hasattr(m, name):
                m.add_module(name, Node())
            m = getattr(m, name)
        m.register_buffer(leaf, value.clone())
    return root


def test_load_clip_model_reads_torchscript_and_state_dict_files(tmp_path):
    from avatarclip_b200.clip_text import load_clip_model
    sd = small_openai_state()
    jit_path, sd_path = str(tmp_path / "ViT-B-32.pt"), str(tmp_path / "state.pt")
    torch.jit.save(torch.jit.script(_module_tree(sd)), jit_path)
    torch.save(sd, sd_path)
    want_visual = {k for k in sd if k.startswith("visual.")}
    want_text = {"token_embedding.weight", "positional_embedding", "ln_final.weight", "ln_final.bias", "text_projection"} | \
        {k for k in sd if k.startswith("transformer.")}
    assert len(want_text) == 5 + 2 * 12
    for path in (jit_path, sd_path):
        visual, text = load_clip_model(path)
        assert set(visual) == want_visual and set(text) == want_text, path
        for k in want_visual | want_text:
            assert torch.equal((visual.get(k) if k in visual else text[k]), sd[k]), (path, k)


def _c_layout(tmp_path, structs):
    """sizeof and offsetof of every field, as gcc lays out include/avc_b200.h."""
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "avc_b200.h"', "int main(void) {"]
    for cname, cls in structs:
        prog.append(f'  printf("S {cname} %zu\\n", sizeof({cname}));')
        for f, *_ in cls._fields_:
            prog.append(f'  printf("F {cname} {f} %zu\\n", offsetof({cname}, {f}));')
    prog += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(prog))
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    return subprocess.check_output([str(exe)], text=True).split("\n")


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_text_ctypes_structures_match_the_c_layout(tmp_path):
    import re
    from avatarclip_b200.clip_text import ClipTextCfg, ClipTextW
    structs = [("avc_clip_text_cfg", ClipTextCfg), ("avc_clip_text_weights", ClipTextW)]
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "avc_b200.h")).read(), flags=re.S)
    for cname, cls in structs:      # same fields in the same order as the header declares them
        body = re.search(r"typedef struct %s\s*\{(.*?)\}\s*%s\s*;" % (cname, cname), hdr, flags=re.S).group(1)
        names = re.findall(r"\**\s*([A-Za-z_]\w*)\s*(?:\[\w+\])?\s*[,;]", body)
        assert [n for n, *_ in cls._fields_] == names, cname
    out = _c_layout(tmp_path, structs)
    for cname, cls in structs:
        assert f"S {cname} {C.sizeof(cls)}" in out, cname
        for f, *_ in cls._fields_:
            assert f"F {cname} {f} {getattr(cls, f).offset}" in out, (cname, f)


def test_init_clip_names_the_missing_model_and_bpe_files(tmp_path, monkeypatch):
    """Without the clip package init_clip reads openai's files: clip_model_path, else $AVC_CLIP_MODEL, else
    ~/.cache/clip/ViT-B-32.pt; the BPE merges next to the model.  A missing file is named in the error."""
    import re
    import sys
    from test_runner import _runner
    monkeypatch.setitem(sys.modules, "clip", None)
    monkeypatch.delenv("AVC_CLIP_MODEL", raising=False)
    monkeypatch.setenv("HOME", str(tmp_path / "home"))
    r = _runner(tmp_path, "cpu", mode="validate")
    with pytest.raises(FileNotFoundError, match=re.escape(str(tmp_path / "home" / ".cache" / "clip" / "ViT-B-32.pt"))):
        r.init_clip()
    missing = str(tmp_path / "nowhere" / "ViT-B-32.pt")
    with pytest.raises(FileNotFoundError, match=re.escape(missing)):
        r.init_clip(clip_model_path=missing)
    model = tmp_path / "models" / "ViT-B-32.pt"
    model.parent.mkdir()
    model.write_bytes(b"")
    monkeypatch.setenv("AVC_CLIP_MODEL", str(model))
    with pytest.raises(FileNotFoundError, match=re.escape(str(model.parent / "bpe_simple_vocab_16e6.txt.gz"))):
        r.init_clip()
    with pytest.raises(FileNotFoundError, match=re.escape(str(tmp_path / "x.txt.gz"))):
        r.init_clip(bpe_path=str(tmp_path / "x.txt.gz"))
    assert r.clip_tower is None
