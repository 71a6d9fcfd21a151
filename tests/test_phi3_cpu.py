"""Cambrian-Phi3 without a GPU: the pinned sliding-window rule and the fp32 oracle against goldens from the unmodified
reference (tests/golden/phi3_*.npz), the state-dict keys, generate()'s host logic through plain-torch kernel stand-ins
(token-exact against the oracle on a prompt longer than the window), every refusal, and the loader."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_emulation  # noqa: E402
from oracle import phi3_oracle as P  # noqa: E402
from test_phi3_gpu import tiny_phi3  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are installed only without a GPU")
GOLD = os.path.join(HERE, "golden")


def _attn_window(q, k, v, *, causal, kmask=None, scale=None, need_lse=False, out=None, window=0):
    """ops.attn_fwd stand-in with the window: fp32 softmax attention under oracle/phi3_oracle.py's mask."""
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    assert causal
    Q = q.float().transpose(1, 2)
    K = k.float().transpose(1, 2).repeat_interleave(nh // nkv, 1)
    V = v.float().transpose(1, 2).repeat_interleave(nh // nkv, 1)
    s = Q @ K.transpose(-1, -2) * (scale if scale is not None else hd ** -0.5)
    allow = P.sliding_mask(Sq, Skv, window, kmask)[:, None]
    p = torch.nan_to_num(torch.softmax(s.masked_fill(~allow, float("-inf")), -1), 0.0)
    o = (p @ V).transpose(1, 2).to(torch.bfloat16).contiguous()
    if out is not None:
        out.copy_(o)
        o = out
    return o


def _install(monkeypatch, calls=None):
    from cambrian_b200 import ops
    ops_emulation.install(monkeypatch)

    def attn(*a, **k):
        if calls is not None:
            calls.append(k.get("window", 0))
        return _attn_window(*a, **k)
    monkeypatch.setattr(ops, "attn_fwd", attn)


def _ocfg(cfg, window="cfg"):
    return dict(num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads,
                num_hidden_layers=cfg.num_hidden_layers, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
                sliding_window=cfg.sliding_window if window == "cfg" else window)


def test_mask_rule_matches_the_reference_golden():
    z = np.load(os.path.join(GOLD, "phi3_mask.npz"))
    am, W = torch.from_numpy(z["attention_mask"]), int(z["window"])
    S = am.shape[1]
    ref = torch.from_numpy(z["mask"])[:, 0] == 0                       # additive mask: 0 = attend
    ours = P.sliding_mask(S, S, W, am)
    live = am.bool()[:, :, None].expand_as(ours)                        # rows of padded queries are never read
    assert torch.equal(ours[live], ref[live])
    assert (ours.sum(-1)[live[..., 0]] <= W).all()                      # W keys at most, the query's own included
    fa = torch.from_numpy(z["mask_flash"])[:, 0] == 0
    assert not torch.equal(fa[live], ref[live])                         # flash-attn's i - j <= W admits one more key


def test_oracle_layer_matches_the_reference_layer():
    from golden.make_golden import seeded_fill
    z = np.load(os.path.join(GOLD, "phi3_layer.npz"))
    m = np.load(os.path.join(GOLD, "phi3_mask.npz"))
    keys = [str(k) for k in z["keys"]]
    shapes = {"self_attn.qkv_proj.weight": (576, 192), "self_attn.o_proj.weight": (192, 192),
              "mlp.gate_up_proj.weight": (512, 192), "mlp.down_proj.weight": (192, 256),
              "input_layernorm.weight": (192,), "post_attention_layernorm.weight": (192,)}
    assert sorted(keys) == sorted(shapes)
    sd = seeded_fill({k: torch.empty(shapes[k]) for k in keys}, 91)
    cfg = dict(num_attention_heads=2, num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=10000.0,
               sliding_window=int(m["window"]))
    am = torch.from_numpy(m["attention_mask"])
    out = P.layer(sd, "", cfg, torch.from_numpy(z["x"]), torch.from_numpy(z["pos"]), am)
    ref = torch.from_numpy(z["out"])
    live = am.bool()
    torch.testing.assert_close(out[live], ref[live], rtol=1e-5, atol=1e-5)


def test_state_dict_keys_are_the_reference_keys():
    cfg, model = tiny_phi3(layers=2)
    z = np.load(os.path.join(GOLD, "phi3_layer.npz"))
    layer_keys = {str(k) for k in z["keys"]}
    want = {"model.embed_tokens.weight", "model.norm.weight", "lm_head.weight"}
    want |= {f"model.layers.{i}.{k}" for i in range(2) for k in layer_keys}
    assert set(model.state_dict()) == want
    lay = model.get_model().layers[0]
    qkv, gu, _, _ = lay._fused()
    assert qkv.data_ptr() == lay.self_attn.qkv_proj.weight.data_ptr()    # the fused layouts are used without copies
    assert gu.data_ptr() == lay.mlp.gate_up_proj.weight.data_ptr()
    from transformers import AutoConfig, AutoModelForCausalLM
    assert type(AutoModelForCausalLM.from_config(AutoConfig.for_model("cambrian_phi3", **{
        k: getattr(cfg, k) for k in ("vocab_size", "hidden_size", "intermediate_size", "num_hidden_layers",
                                     "num_attention_heads", "sliding_window", "pad_token_id")}))).__name__ == \
        "CambrianPhi3ForCausalLM"


@needs_no_gpu
@pytest.mark.parametrize("padded", [False, True])
def test_greedy_generate_host_logic_matches_oracle(monkeypatch, padded):
    calls = []
    _install(monkeypatch, calls)
    cfg, model = tiny_phi3(window=7, layers=2)
    model = model.to(torch.bfloat16)
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    ids = torch.randint(3, cfg.vocab_size, (2, 12), generator=torch.Generator().manual_seed(4))
    am = torch.ones_like(ids)
    if padded:
        am[1, :4] = 0
    n_new = 10                                                   # prompt 12 > W = 7; 10 more positions past it
    got = model.generate(ids, attention_mask=am, max_new_tokens=n_new, do_sample=False, eos_token_id=None)
    assert set(calls) == {7}                                      # every attention call carries the window
    want, margins = P.greedy(sd, _ocfg(cfg), ids, n_new, attention_mask=am)
    assert got.tolist() == want, (got.tolist(), want, margins)
    assert min(margins) > 0.5, margins


@needs_no_gpu
def test_stopping_criterion_and_eos(monkeypatch):
    _install(monkeypatch)
    cfg, model = tiny_phi3(window=7, layers=2)
    model = model.to(torch.bfloat16)
    ids = torch.randint(3, cfg.vocab_size, (1, 12), generator=torch.Generator().manual_seed(4))
    full = model.generate(ids, max_new_tokens=10, do_sample=False, eos_token_id=None)
    stop_at = int(full[0, 3])
    got = model.generate(ids, max_new_tokens=10, do_sample=False, eos_token_id=stop_at)
    assert got[0].tolist() == full[0, :full[0].tolist().index(stop_at) + 1].tolist()
    seen = []
    got = model.generate(ids, max_new_tokens=10, do_sample=False, eos_token_id=None,
                         stopping_criteria=[lambda g, s: seen.append(g.shape[1]) or g.shape[1] >= 5])
    assert got.shape[1] == 5 and torch.equal(got, full[:, :5])


def test_refusals():
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3Config, CambrianPhi3ForCausalLM
    cfg, model = tiny_phi3(layers=1)
    with pytest.raises(NotImplementedError, match="Phi3.*backward"):
        model(input_ids=torch.zeros(1, 4, dtype=torch.long))
    from cambrian_b200.engine import TrainEngine
    with pytest.raises(NotImplementedError, match="Phi3.*backward"):
        TrainEngine(model)
    from cambrian_b200.sharded import Zero3Inference
    with pytest.raises(NotImplementedError, match="Zero3Inference.*Phi3"):
        Zero3Inference(model)
    with pytest.raises(NotImplementedError, match="Phi3.*fp8.*96"):
        model.generate(torch.zeros(1, 4, dtype=torch.long), kv_cache_dtype="fp8")
    for kind, extra in (("su", {}), ("yarn", {"factor": 32.0})):
        with pytest.raises(NotImplementedError, match=f"Phi3.*{kind}"):
            CambrianPhi3ForCausalLM(CambrianPhi3Config(
                vocab_size=64, hidden_size=192, intermediate_size=256, num_hidden_layers=1, num_attention_heads=2,
                pad_token_id=0, rope_scaling=dict(type=kind, short_factor=[1.0] * 48, long_factor=[1.0] * 48, **extra)))


@pytest.mark.parametrize("flag", ["load_4bit", "load_8bit", "load_fp8"])
def test_loader_refuses_quantised_phi3(flag):
    from cambrian_b200 import checkpoint
    with pytest.raises(NotImplementedError, match=f"Phi3 with {flag}"):
        checkpoint.load_pretrained_model("x", model_name="cambrian-phi3-3b", device="cpu", load_tokenizer=False,
                                         **{flag: True})


def test_loader_builds_phi3_from_a_saved_directory(tmp_path):
    from cambrian_b200 import checkpoint
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3ForCausalLM
    cfg, model = tiny_phi3(layers=2)
    model.save_pretrained(tmp_path)
    _, loaded, procs, ctx = checkpoint.load_pretrained_model(str(tmp_path), model_name="cambrian-phi3-3b",
                                                             device="cpu", load_tokenizer=False)
    assert isinstance(loaded, CambrianPhi3ForCausalLM) and procs == []
    assert loaded.config.sliding_window == cfg.sliding_window
    for k, v in model.state_dict().items():
        assert torch.equal(loaded.state_dict()[k].float(), v.to(torch.bfloat16).float()), k
