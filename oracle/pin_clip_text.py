"""Cross-check the restated CLIP text tower (oracle/clip_text.py) against the independent HuggingFace ``transformers``
implementation of the same published architecture (``CLIPTextModelWithProjection``), on seeded random weights (the
real ViT-B-32.pt is not on disk).  Like oracle/pin_clip.py this validates the restatement of the ARCHITECTURE; parity
with openai/CLIP's own code stays unpinned.

HF pools at the first position of ``eos_token_id`` (49407, the default) and openai at ``argmax(tokens)``: the token
rows here end in 49407, the largest id, so both pick the same row.

    python -m oracle.pin_clip_text
"""
import torch


def sample_tokens(conf, eot_positions, seed=0):
    """Rows <|startoftext|> (vocab-2), random ids, <|endoftext|> (vocab-1) at the given position, zeros after it."""
    g = torch.Generator().manual_seed(seed)
    tok = torch.zeros(len(eot_positions), conf.context, dtype=torch.int32)
    for i, e in enumerate(eot_positions):
        tok[i, 0] = conf.vocab - 2
        tok[i, 1:e] = torch.randint(1, conf.vocab - 2, (e - 1,), generator=g, dtype=torch.int32)
        tok[i, e] = conf.vocab - 1
    return tok


def main():
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    from oracle import clip_text as ct

    conf = ct.TextConf()
    sd = ct.random_text_state(conf, seed=0)
    cfg = CLIPTextConfig(vocab_size=conf.vocab, hidden_size=conf.width, intermediate_size=conf.mlp,
                         num_hidden_layers=conf.layers, num_attention_heads=conf.heads,
                         max_position_embeddings=conf.context, hidden_act="quick_gelu", projection_dim=conf.out_dim,
                         layer_norm_eps=1e-5)
    assert cfg.eos_token_id == conf.vocab - 1, cfg.eos_token_id
    hf = CLIPTextModelWithProjection(cfg).eval()
    m = hf.state_dict()
    W = conf.width

    def put(k, v):
        assert m[k].shape == v.shape, (k, m[k].shape, v.shape)
        m[k] = v.clone()

    put("text_model.embeddings.token_embedding.weight", sd["token_embedding.weight"])
    put("text_model.embeddings.position_embedding.weight", sd["positional_embedding"])
    put("text_model.final_layer_norm.weight", sd["ln_final.weight"])
    put("text_model.final_layer_norm.bias", sd["ln_final.bias"])
    for i in range(conf.layers):
        p, q = f"transformer.resblocks.{i}.", f"text_model.encoder.layers.{i}."
        for a, b in (("layer_norm1", "ln_1"), ("layer_norm2", "ln_2")):
            put(q + a + ".weight", sd[p + b + ".weight"]); put(q + a + ".bias", sd[p + b + ".bias"])
        wi, bi = sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"]
        for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
            put(q + f"self_attn.{n}.weight", wi[j * W:(j + 1) * W]); put(q + f"self_attn.{n}.bias", bi[j * W:(j + 1) * W])
        put(q + "self_attn.out_proj.weight", sd[p + "attn.out_proj.weight"])
        put(q + "self_attn.out_proj.bias", sd[p + "attn.out_proj.bias"])
        put(q + "mlp.fc1.weight", sd[p + "mlp.c_fc.weight"]); put(q + "mlp.fc1.bias", sd[p + "mlp.c_fc.bias"])
        put(q + "mlp.fc2.weight", sd[p + "mlp.c_proj.weight"]); put(q + "mlp.fc2.bias", sd[p + "mlp.c_proj.bias"])
    put("text_projection.weight", sd["text_projection"].t().contiguous())
    hf.load_state_dict(m)

    tok = sample_tokens(conf, [3, 40, 76], seed=1)
    with torch.no_grad():
        a = ct.encode_text(sd, tok, conf)
        b = hf(input_ids=tok.long()).text_embeds
    err = (a - b).abs().max().item() / b.abs().max().item()
    print(f"[pin_clip_text] restated text tower vs transformers CLIPTextModelWithProjection: rel-to-max err {err:.2e}")
    assert err < 1e-4
    return err


if __name__ == "__main__":
    main()
