import json
import os
import re

import pytest
import torch

from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM, build_model, preset


def tiny_llama(**kw):
    cfg = dict(vocab_size=131, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=4,
               num_key_value_heads=2, max_position_embeddings=64, pad_vocab_multiple=16)
    cfg.update(kw)
    return LlamaForCausalLM(LlamaConfig(**cfg))


# parameter and checkpoint layout of tiny native models ({llama, gpt_neo} x {tied, untied}): the flat arena, optimizer shards and
# elastic resume follow named_parameters(); checkpoint files follow state_dict()
with open(os.path.join(os.path.dirname(__file__), "golden", "native_checkpoint_layout.json")) as _f:
    LAYOUT = json.load(_f)
# HF buffers a checkpoint may carry that have no parameter here
HF_BUFFERS = {"llama": ["model.layers.0.self_attn.rotary_emb.inv_freq"],
              "gpt_neo": ["transformer.h.0.attn.attention.bias", "transformer.h.0.attn.attention.masked_bias"]}


def native(case, seed=0):
    cls, cfg = {"llama": (LlamaForCausalLM, LlamaConfig), "gpt_neo": (GPTForCausalLM, GPTConfig)}[case.rsplit("_", 1)[0]]
    torch.manual_seed(seed)
    return cls(cfg(**LAYOUT[case]["config"])).float()


@pytest.mark.parametrize("case", list(LAYOUT))
def test_native_layout_matches_golden(case):
    m = native(case)
    assert [[n, list(p.shape)] for n, p in m.named_parameters()] == LAYOUT[case]["named_parameters"]
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == LAYOUT[case]["state_dict"]


@pytest.mark.parametrize("case", list(LAYOUT))
def test_native_checkpoint_roundtrip(case):
    src, dst = native(case, seed=1), native(case, seed=0)
    assert dst.load_state_dict({k: v.clone() for k, v in src.state_dict().items()}) == ([], [])
    for (name, p), q in zip(dst.named_parameters(), src.parameters()):
        assert torch.equal(p, q), name                        # vocabulary padding rows included: zero in both
    # saved tensors are views of the live parameters, under DDP's prefix too
    sd = dst.state_dict(prefix="module.", keep_vars=True)
    assert list(sd) == ["module." + k for k, _ in LAYOUT[case]["state_dict"]] and all(v.requires_grad for v in sd.values())
    with torch.no_grad():
        dst.head_weight[0, 0] = 5.0
    assert dst.state_dict()["lm_head.weight"][0, 0] == 5.0


@pytest.mark.parametrize("case", list(LAYOUT))
def test_native_load_strict(case):
    m = native(case)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(RuntimeError, match=re.escape("unexpected=['bogus.weight']")):
        m.load_state_dict({**sd, "bogus.weight": torch.zeros(1)})
    first = next(iter(sd))
    less = {k: v for k, v in sd.items() if k != first}
    with pytest.raises(RuntimeError, match=re.escape(f"missing=['{first}']")):
        m.load_state_dict(less)
    assert m.load_state_dict({**less, "bogus.weight": torch.zeros(1)}, strict=False) == ([first], ["bogus.weight"])


@pytest.mark.parametrize("case", list(LAYOUT))
def test_native_load_ignores_own_hf_buffers(case):
    family = case.rsplit("_", 1)[0]
    other = HF_BUFFERS["gpt_neo" if family == "llama" else "llama"]
    m = native(case)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    assert m.load_state_dict({**sd, **{k: torch.zeros(1) for k in HF_BUFFERS[family]}}) == ([], [])
    assert m.load_state_dict({**sd, **{k: torch.zeros(1) for k in other}}, strict=False) == ([], other)


@pytest.mark.parametrize("case", list(LAYOUT))
def test_native_load_lm_head(case):
    """A tied head is the embedding: it neither needs ``lm_head.weight`` nor reports it, and ignores its values."""
    tied = case.endswith("_tied")
    m = native(case)
    sd = {k: v.clone() for k, v in native(case, seed=1).state_dict().items()}
    sd.pop("lm_head.weight")
    assert m.load_state_dict(sd, strict=False) == ([] if tied else ["lm_head.weight"], [])
    if not tied:
        with pytest.raises(RuntimeError, match=re.escape("missing=['lm_head.weight']")):
            m.load_state_dict(sd)
    embed = next(iter(sd))
    assert m.load_state_dict({**sd, "lm_head.weight": torch.zeros_like(sd[embed])}) == ([], [])
    head = m.state_dict()["lm_head.weight"]
    assert torch.equal(head, sd[embed]) if tied else not head.any()


def test_llama_param_count_presets():
    assert LlamaConfig.from_dict(dict(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16,
                                      num_attention_heads=32, num_key_value_heads=8, tie_word_embeddings=True)).num_parameters() == 1_235_814_400
    assert LlamaConfig.from_dict(dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                                      num_attention_heads=32, num_key_value_heads=8, tie_word_embeddings=False)).num_parameters() == 8_030_261_248
    m = preset("tiny")
    assert m.num_parameters() == m.config.num_parameters(padded=True)


@pytest.mark.parametrize("tied", [True, False])
def test_llama_matches_hf(tied):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(0)
    mine = tiny_llama(tie_word_embeddings=tied).float()
    c = mine.config
    hf_cfg = transformers.LlamaConfig(
        vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
        num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
        num_key_value_heads=c.num_key_value_heads, max_position_embeddings=c.max_position_embeddings,
        rms_norm_eps=c.rms_norm_eps, rope_theta=c.rope_theta, tie_word_embeddings=tied, attention_bias=False,
        mlp_bias=False, attn_implementation="eager")
    hf = transformers.LlamaForCausalLM(hf_cfg).float().eval()
    # our checkpoint -> HF model: key names and shapes must be HF's
    sd = {k: v.clone() for k, v in mine.state_dict().items()}
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in k for k in missing)
    ids = torch.randint(0, c.vocab_size, (2, 17))
    ref = hf(input_ids=ids, labels=ids)
    out = mine(input_ids=ids, labels=ids)
    torch.testing.assert_close(out[0], ref.loss, rtol=1e-4, atol=1e-5)
    logits = mine(input_ids=ids).logits
    torch.testing.assert_close(logits, ref.logits, rtol=1e-3, atol=1e-4)
    # gradients agree too (through the fused-accumulation linear / embedding paths)
    out[0].backward()
    ref.loss.backward()
    g_mine = mine.model.layers[0].mlp.down_proj.grad
    g_ref = hf.model.layers[0].mlp.down_proj.weight.grad
    torch.testing.assert_close(g_mine, g_ref, rtol=1e-3, atol=1e-5)
    ge = mine.model.embed_tokens.grad[: c.vocab_size]
    ge_ref = hf.model.embed_tokens.weight.grad
    torch.testing.assert_close(ge, ge_ref, rtol=1e-3, atol=1e-5)
    assert mine.model.embed_tokens.grad[c.vocab_size:].abs().sum() == 0     # vocab padding gets no gradient
    # and HF -> ours
    mine2 = tiny_llama(tie_word_embeddings=tied).float()
    mine2.load_state_dict(hf.state_dict())
    torch.testing.assert_close(mine2(input_ids=ids, labels=ids)[0], ref.loss.detach(), rtol=1e-4, atol=1e-5)


def test_llama_labels_ignore_index():
    torch.manual_seed(0)
    m = tiny_llama().float()
    ids = torch.randint(0, 131, (2, 12))
    labels = ids.clone()
    labels[:, 6:] = -100
    l1 = m(input_ids=ids, labels=labels)[0]
    ids2 = ids.clone()
    ids2[:, 7:] = 5       # tokens after the last supervised position cannot matter (causal)
    l2 = m(input_ids=ids2, labels=labels)[0]
    torch.testing.assert_close(l1, l2)


def test_gptneo_matches_hf():
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(0)
    cfg = GPTConfig(vocab_size=97, hidden_size=32, num_hidden_layers=4, num_attention_heads=4, max_position_embeddings=40,
                    attention_layers="alternating", window_size=8, scale_attn=False)
    mine = GPTForCausalLM(cfg).float()
    hf_cfg = transformers.GPTNeoConfig(vocab_size=97, hidden_size=32, num_layers=4, num_heads=4, max_position_embeddings=40,
                                       attention_types=[[["global", "local"], 2]], window_size=8, intermediate_size=128,
                                       attention_dropout=0, embed_dropout=0, resid_dropout=0, attn_implementation="eager")
    hf = transformers.GPTNeoForCausalLM(hf_cfg).float().eval()
    missing, unexpected = hf.load_state_dict(mine.state_dict(), strict=False)
    assert not unexpected, unexpected
    assert all(k.endswith(("attn.attention.bias", "masked_bias")) for k in missing), missing
    ids = torch.randint(0, 97, (2, 33))
    ref = hf(input_ids=ids, labels=ids)
    out = mine(input_ids=ids, labels=ids)
    torch.testing.assert_close(out[0], ref.loss, rtol=1e-4, atol=1e-5)
    mine.load_state_dict(hf.state_dict())


def test_gptneo_json_config_roundtrip():
    import acco_b200.config as C
    cfg = C.compose(overrides=["model=gptneo"])
    m = build_model(dict(cfg.model, num_hidden_layers=None) if False else cfg.model, config_root=None)
    assert isinstance(m, GPTForCausalLM)
    assert m.config.attention_layers == ["global", "local"] * 6 and m.config.window_size == 256 and not m.config.scale_attn
    assert m.num_parameters() == 124_412_160 + 0   # reference model size minus nothing: wte 38.6M + wpe 0.79M + 12 blocks
    g = build_model(C.compose(overrides=["model=gpt2-small"]).model)
    assert g.config.scale_attn and set(g.config.attention_layers) == {"global"}


def test_output_indexing():
    m = tiny_llama().float()
    ids = torch.randint(0, 131, (1, 5))
    o = m(input_ids=ids, labels=ids)
    assert o[0] is o.loss and o["loss"] is o.loss and list(o.keys()) == ["loss"]
    o2 = m(input_ids=ids)
    assert o2[0] is o2.logits and o2.logits.shape == (1, 5, 131)


@pytest.mark.parametrize("family", ["llama", "llama3-rope", "gpt_neo", "other"])
def test_from_pretrained_hf_directory(tmp_path, family):
    """`main.py model.pretrained=<dir>`: an HF `save_pretrained` directory (config.json + safetensors) loads into the native
    model when the architecture has one (same logits as the HF module), else falls back to the HF module like the reference."""
    transformers = pytest.importorskip("transformers")
    from acco_b200.models import from_pretrained
    torch.manual_seed(0)
    if family.startswith("llama"):
        rs = dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0, original_max_position_embeddings=32) \
            if family == "llama3-rope" else None
        hf = transformers.LlamaForCausalLM(transformers.LlamaConfig(
            vocab_size=131, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
            max_position_embeddings=64, tie_word_embeddings=False, rope_scaling=rs, attn_implementation="eager"))
        want = LlamaForCausalLM
    elif family == "gpt_neo":
        hf = transformers.GPTNeoForCausalLM(transformers.GPTNeoConfig(
            vocab_size=97, hidden_size=32, num_layers=2, num_heads=4, max_position_embeddings=40, attention_types=[[["global", "local"], 1]],
            window_size=8, intermediate_size=128, attention_dropout=0, embed_dropout=0, resid_dropout=0, attn_implementation="eager"))
        want = GPTForCausalLM
    else:
        hf = transformers.GPT2LMHeadModel(transformers.GPT2Config(vocab_size=97, n_embd=32, n_layer=1, n_head=2, n_positions=40))
        want = transformers.GPT2LMHeadModel
    hf = hf.float().eval()
    hf.save_pretrained(tmp_path / "ck")
    m = from_pretrained(str(tmp_path / "ck"))
    assert isinstance(m, want)
    ids = torch.randint(0, 90, (2, 21))
    ref = hf(input_ids=ids, labels=ids)
    out = m(input_ids=ids, labels=ids)
    torch.testing.assert_close(out[0], ref.loss, rtol=1e-4, atol=1e-5)


def test_cli_finetune_from_pretrained_directory(tmp_path, monkeypatch):
    """End to end through main.py: `train=acco-ft model.pretrained=<HF dir>` finetunes the loaded weights (reference `main.py:33-35`)."""
    transformers = pytest.importorskip("transformers")
    import sys
    torch.manual_seed(0)
    hf = transformers.LlamaForCausalLM(transformers.LlamaConfig(
        vocab_size=260, hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=4, num_key_value_heads=2,
        max_position_embeddings=64, tie_word_embeddings=True, attn_implementation="eager"))
    hf.save_pretrained(tmp_path / "ck")
    root = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))
    sys.path.insert(0, root)
    import main as cli
    monkeypatch.chdir(tmp_path)
    stats = cli.main(["train=acco-ft", "data=alpaca", "model=tiny", f"model.pretrained={tmp_path / 'ck'}", "data.synthetic=true",
                      "data.synthetic_docs=64", "data.synthetic_mean_len=20", "train.nb_steps_tot=4", "train.batch_size=2", "train.max_length=32",
                      "train.save=False", "train.tensorboard=False", "train.use_mixed_precision=False"])
    assert stats["count_grad_tot"] >= 4
