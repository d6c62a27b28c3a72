"""CLIP text tower, host side (no GPU): the tokenizer against transformers' CLIPTokenizer, the CPU oracle against
transformers' CLIPTextModelWithProjection, the weight loader, SRC_TRG_TXT_DIC parsing and the CLI surface."""
import argparse
import json
import os

import pytest
import torch

from asyrp_official_b200 import clip_text, synthetic
from oracle import clip_text as oct

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROMPTS = ["face", "smiling face", "Person with Blond hair", "a photo of the person's   face, 2 cats & 13 dogs!",
           "self-portrait by Frida Kahlo", "  tanned\tface  ", "painting by Gogh", "it's we'll they're I'd"]
UNSEEN = ["zebra crossing at dusk", "café au lait"]  # words the synthetic merges do not build whole


@pytest.fixture
def vocab(tmp_path):
    """a synthetic bpe .txt.gz, and transformers' vocab.json / merges.txt holding the same vocabulary"""
    merges = synthetic.clip_bpe_merges(PROMPTS)
    gz = str(tmp_path / "bpe.txt.gz")
    n = synthetic.write_clip_vocab(gz, merges)
    syms = list(oct.bytes_to_unicode().values())
    words = syms + [s + "</w>" for s in syms] + ["".join(m) for m in merges] + ["<|startoftext|>", "<|endoftext|>"]
    assert len(words) == n
    (tmp_path / "vocab.json").write_text(json.dumps({w: i for i, w in enumerate(words)}))
    (tmp_path / "merges.txt").write_text("\n".join(["#version: 0.2"] + [f"{a} {b}" for a, b in merges]) + "\n")
    return gz, str(tmp_path / "vocab.json"), str(tmp_path / "merges.txt"), n


def test_tokenizer_matches_transformers_and_the_oracle(vocab):
    from transformers import CLIPTokenizer
    gz, vj, mt, n = vocab
    tok = clip_text.Tokenizer(gz)
    assert len(tok) == n and tok.eot == n - 1 and tok.sot == n - 2
    hf = CLIPTokenizer(vj, mt)
    ref = oct.SimpleTokenizer(gz)
    for p in PROMPTS + UNSEEN:
        ids = tok.tokenize(p)[0]
        k = int(ids.argmax()) + 1  # up to EOT; CLIP pads with 0, transformers with EOT
        assert ids[k:].eq(0).all()
        assert ids[:k].tolist() == hf(p)["input_ids"], p
        assert torch.equal(ids, ref.tokenize([p])[0]), p
    # whole words of the merges are one token each
    assert tok.encode("smiling face") == [tok.encoder["smiling</w>"], tok.encoder["face</w>"]]


def test_tokenizer_cleaning_and_batch(vocab):
    gz = vocab[0]
    tok, ref = clip_text.Tokenizer(gz), oct.SimpleTokenizer(gz)
    for p in ["Cats &amp;amp; Dogs", "FACE\n\nface", "&lt;b&gt;face"]:  # html.unescape twice, whitespace, case
        assert torch.equal(tok.tokenize(p), ref.tokenize([p])), p
    assert tok.encode("Cats &amp;amp; Dogs") == tok.encode("cats & dogs")
    assert tok.tokenize(PROMPTS).shape == (len(PROMPTS), 77) and tok.tokenize(PROMPTS).dtype == torch.long


def test_tokenizer_rejects_a_prompt_that_is_too_long(vocab):
    tok = clip_text.Tokenizer(vocab[0])
    assert tok.tokenize(" ".join(["face"] * 75))[0, 76] == tok.eot  # 75 + SOT + EOT fits exactly
    with pytest.raises(RuntimeError, match="too long"):
        tok.tokenize(" ".join(["face"] * 76))


def _hf_state_dict(sd, layers):
    """CLIP's text-tower keys -> transformers' CLIPTextModelWithProjection keys"""
    out = {"text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
           "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
           "text_model.final_layer_norm.weight": sd["ln_final.weight"],
           "text_model.final_layer_norm.bias": sd["ln_final.bias"],
           "text_projection.weight": sd["text_projection"].t()}
    for i in range(layers):
        c, h = f"transformer.resblocks.{i}.", f"text_model.encoder.layers.{i}."
        for a, b in (("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("attn.out_proj", "self_attn.out_proj"),
                     ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            out[h + b + ".weight"], out[h + b + ".bias"] = sd[c + a + ".weight"], sd[c + a + ".bias"]
        for part, q in zip(sd[c + "attn.in_proj_weight"].chunk(3), "qkv"):
            out[h + f"self_attn.{q}_proj.weight"] = part
        for part, q in zip(sd[c + "attn.in_proj_bias"].chunk(3), "qkv"):
            out[h + f"self_attn.{q}_proj.bias"] = part
    return out


def test_oracle_matches_transformers_clip_text_model(vocab):
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    gz, _, _, n = vocab
    width, layers, embed = 128, 3, 64
    sd = synthetic.clip_text_state_dict(seed=3, width=width, layers=layers, vocab=n, embed_dim=embed)
    cfg = CLIPTextConfig(vocab_size=n, hidden_size=width, intermediate_size=4 * width, num_hidden_layers=layers,
                         num_attention_heads=width // 64, max_position_embeddings=77, projection_dim=embed,
                         hidden_act="quick_gelu", layer_norm_eps=1e-5, eos_token_id=n - 1, bos_token_id=n - 2,
                         pad_token_id=0)
    model = CLIPTextModelWithProjection(cfg).eval()
    missing, unexpected = model.load_state_dict(_hf_state_dict(sd, layers), strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    ids = clip_text.Tokenizer(gz).tokenize(PROMPTS)
    with torch.no_grad():
        ref = model(input_ids=ids).text_embeds
        out = oct.encode_text(sd, ids, dtype=torch.float32)
    e = (out - ref).abs().max().item() / ref.abs().max().item()
    assert e <= 1e-5, e
    c = oct.cosine(out[:4], out[4:])
    assert torch.allclose(c, torch.nn.functional.cosine_similarity(ref[:4], ref[4:], dim=1, eps=1e-6), atol=1e-5)


def test_synthetic_weights_have_no_zero_term():
    sd = synthetic.clip_text_state_dict(seed=1, width=64, layers=2, vocab=600, embed_dim=64)
    assert set(sd) == set(clip_text.text_key_shapes(64, 2, 77, 600, 64))
    for k, v in sd.items():
        assert v.dtype == torch.float32 and (v != 0).all(), k
    assert (sd["ln_final.bias"].abs().max() > 0) and not torch.equal(sd["ln_final.weight"], torch.ones(64))
    assert torch.equal(sd["ln_final.bias"], synthetic.clip_text_state_dict(seed=1, width=64, layers=2, vocab=600,
                                                                           embed_dim=64)["ln_final.bias"])


class _Holder(torch.nn.Module):
    def forward(self, x):
        return x


def _jit_archive(sd, path):
    """a TorchScript archive whose state_dict() is sd, as CLIP's downloaded ViT-B-16.pt is"""
    root = _Holder()
    for name, t in sd.items():
        *mods, leaf = name.split(".")
        m = root
        for part in mods:
            if not hasattr(m, part):
                m.add_module(part, _Holder())
            m = getattr(m, part)
        m.register_buffer(leaf, t)
    torch.jit.save(torch.jit.script(root), path)


def _full_clip(seed=2, width=64, layers=2, vocab=600, embed=64):
    sd = synthetic.clip_text_state_dict(seed=seed, width=width, layers=layers, vocab=vocab, embed_dim=embed)
    sd = {k: v.half() for k, v in sd.items()}  # CLIP stores its weights in fp16
    sd.update({"visual.conv1.weight": torch.randn(8, 3, 4, 4).half(), "visual.proj": torch.randn(8, embed).half(),
               "logit_scale": torch.tensor(4.6), "input_resolution": torch.tensor(224),
               "context_length": torch.tensor(77), "vocab_size": torch.tensor(vocab)})
    return sd


def test_loader_reads_a_torchscript_archive_and_a_state_dict(tmp_path):
    sd = _full_clip()
    _jit_archive(sd, str(tmp_path / "ViT-B-16.pt"))
    torch.save(sd, tmp_path / "plain.pth")
    for src in (str(tmp_path / "ViT-B-16.pt"), str(tmp_path / "plain.pth"), sd):
        dims, t = clip_text.load_state_dict(src, vocab_size=600)
        assert dims == dict(width=64, heads=1, layers=2, context=77, vocab=600, embed_dim=64)
        assert set(t) == set(clip_text.text_key_shapes(64, 2, 77, 600, 64))
        assert all(v.dtype == torch.float32 for v in t.values())
        assert torch.equal(t["ln_final.bias"], sd["ln_final.bias"].float())
    dims, _ = clip_text.load_state_dict(synthetic.clip_text_state_dict(width=128, layers=3, vocab=600, embed_dim=192))
    assert (dims["heads"], dims["layers"], dims["embed_dim"]) == (2, 3, 192)


def test_loader_rejects_bad_state_dicts():
    sd = _full_clip()
    cases = {"missing": {k: v for k, v in sd.items() if k != "transformer.resblocks.1.mlp.c_fc.bias"},
             "missing_top": {k: v for k, v in sd.items() if k != "ln_final.bias"},
             "shape": {**sd, "transformer.resblocks.0.attn.in_proj_weight": torch.zeros(3 * 64, 32)},
             "shape_pos": {**sd, "positional_embedding": torch.zeros(77, 32)},
             "unknown": {**sd, "transformer.resblocks.0.attn.extra": torch.zeros(2)},
             "unknown_top": {**sd, "text_bias": torch.zeros(2)}}
    for what, bad in cases.items():
        with pytest.raises(ValueError):
            clip_text.load_state_dict(bad)
            pytest.fail(what)
    with pytest.raises(ValueError, match="vocabulary"):
        clip_text.load_state_dict(sd, vocab_size=601)


def test_text_dic_is_parsed_not_executed(tmp_path):
    from asyrp_official_b200.diffusion_latent import read_text_dic
    p = tmp_path / "text_dic.py"
    p.write_text("import module_that_does_not_exist\n"
                 "SRC_TRG_TXT_DIC = {\n    # faces\n    'smiling': (['face'],\n                ['smiling face']),\n"
                 "    'old': (['person'], ['old person']),\n}\nraise SystemExit(1)\n")
    dic = read_text_dic(str(p))
    assert dic == {"smiling": (["face"], ["smiling face"]), "old": (["person"], ["old person"])}
    (tmp_path / "empty.py").write_text("OTHER = 1\n")
    with pytest.raises(ValueError):
        read_text_dic(str(tmp_path / "empty.py"))
    with pytest.raises(FileNotFoundError):
        read_text_dic(str(tmp_path / "nope.py"))


def test_cli_flags_and_edit_texts(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    os.makedirs("utils")
    with open("utils/text_dic.py", "w") as f:
        f.write("SRC_TRG_TXT_DIC = {'smiling': (['face'], ['smiling face'])}\n")
    with open("other_dic.py", "w") as f:
        f.write("SRC_TRG_TXT_DIC = {'smiling': (['a face'], ['a smiling face'])}\n")
    args, cfg = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml", "--edit_attr", "smiling",
                                           "--clip_weights", "w.pt", "--clip_vocab", "v.txt.gz"])
    assert (args.clip_weights, args.clip_vocab, args.text_dic, args.src_txts) == ("w.pt", "v.txt.gz", None, None)
    r = Asyrp(args, cfg, device="cpu")
    assert r.clip_configured() and r.needs_clip()
    assert r.edit_texts() == (["face"], ["smiling face"])
    args.text_dic = "other_dic.py"
    assert r.edit_texts() == (["a face"], ["a smiling face"])
    with pytest.raises(ValueError):
        r.edit_texts("frowning")
    with pytest.raises(ValueError):
        r.edit_texts("attribute")
    args, cfg = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml", "--src_txts", "face", "--trg_txts",
                                           "old face", "--src_txts", "x", "--trg_txts", "y", "--clip_cosine", "0.5"])
    r = Asyrp(args, cfg, device="cpu")
    assert args.edit_attr is None and r.edit_texts() == (["face", "x"], ["old face", "y"]) and not r.needs_clip()


def test_without_any_t_edit_source_the_runner_still_raises(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    args, cfg = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml", "--edit_attr", "smiling",
                                           "--lpips_table_dir", os.path.join(ROOT, "tests", "golden", "lpips")])
    with pytest.raises(ValueError, match="--clip_weights and --clip_vocab"):
        Asyrp(args, cfg, device="cpu").set_t_edit_t_addnoise()
    args.clip_weights = "w.pt"  # half of the CLIP pair is not enough
    with pytest.raises(ValueError, match="--clip_weights and --clip_vocab"):
        Asyrp(args, cfg, device="cpu").set_t_edit_t_addnoise()
    a = argparse.Namespace(user_defined_t_edit=None, user_defined_t_addnoise=None, edit_attr="smiling",
                           clip_weights="w.pt", clip_vocab="v.gz")
    with pytest.raises(ValueError):  # no LPIPS table
        Asyrp(a, cfg, device="cpu").set_t_edit_t_addnoise()
