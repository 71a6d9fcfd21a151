"""Cambrian-Phi3 training without a GPU: the differentiable restatement of the fp32 oracle (tests/phi3_train_reference.py)
against the oracle's forward and against the reference's Phi3DecoderLayer gradients (tests/golden/phi3_layer_grad.npz),
and the host logic of training a tiny Phi-3 (head dim 96, a window shorter than the sequence, right padding whose last
queries see no key) through plain-torch kernel stand-ins: loss and every parameter gradient against that reference, the
window on both attention calls of every layer, recompute, the fused leaves' gradients under plain autograd and in
TrainEngine's main_grad, and the training refusals."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_emulation  # noqa: E402
import phi3_train_reference as R  # noqa: E402
from oracle import phi3_oracle as P  # noqa: E402
from test_phi3_gpu import tiny_phi3  # noqa: E402

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are installed only without a GPU")
GOLD = os.path.join(HERE, "golden")
W, S, VALID = 5, 12, 7          # the second row has VALID tokens: at W = 5 its query slots 11.. see no key


def _install(monkeypatch, calls):
    """ops_emulation, with its attn_fwd / attn_bwd wrapped to record the window of every call; the CUDA-bf16 training
    guard is lifted so the CPU model trains."""
    from cambrian_b200 import ops
    from cambrian_b200.model.language_model import cambrian_phi3
    ops_emulation.install(monkeypatch)
    monkeypatch.setattr(cambrian_phi3, "require_cuda_bf16", lambda model: None)

    def recording(kind, fn):
        def wrapped(*args, causal, window=0, **kw):
            assert causal
            calls.append((kind, window))
            return fn(*args, causal=causal, window=window, **kw)
        return wrapped

    monkeypatch.setattr(ops, "attn_fwd", recording("fwd", ops_emulation.attn_fwd))
    monkeypatch.setattr(ops, "attn_bwd", recording("bwd", ops_emulation.attn_bwd))


def _batch(vocab):
    ids = torch.randint(3, vocab, (2, S), generator=torch.Generator().manual_seed(21))
    am = torch.ones(2, S, dtype=torch.long)
    am[1, VALID:] = 0                                             # right padding, as training batches are
    labels = ids.masked_fill(am == 0, -100)
    return ids, am, labels


def _model(layers=2):
    cfg, model = tiny_phi3(window=W, layers=layers)
    with torch.no_grad():                                         # a tamer test model than tiny_phi3's decode one
        for n, p in model.named_parameters():
            if n.endswith("o_proj.weight"):
                p.div_(15.0)
    return cfg, model.to(torch.bfloat16).train()


def _oracle_loss_and_grads(model, cfg, ids, am, labels):
    sd = {k: v.detach().float().requires_grad_() for k, v in model.state_dict().items()}
    ocfg = dict(num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads,
                num_hidden_layers=cfg.num_hidden_layers, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
                sliding_window=cfg.sliding_window)
    lg = R.logits(sd, ocfg, ids, kmask=am)
    loss = torch.nn.functional.cross_entropy(lg[:, :-1].reshape(-1, lg.shape[-1]), labels[:, 1:].reshape(-1),
                                             ignore_index=-100)
    loss.backward()
    return loss.item(), {k: v.grad for k, v in sd.items()}


def _grads(model):
    return {n: p.grad.detach().float().clone() for n, p in model.named_parameters()}


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


SHAPES = {"self_attn.qkv_proj.weight": (576, 192), "self_attn.o_proj.weight": (192, 192),
          "mlp.gate_up_proj.weight": (512, 192), "mlp.down_proj.weight": (192, 256),
          "input_layernorm.weight": (192,), "post_attention_layernorm.weight": (192,)}


def test_training_reference_matches_the_oracle_forward_and_the_reference_gradients():
    from golden.make_golden import seeded_fill
    z = np.load(os.path.join(GOLD, "phi3_layer_grad.npz"))
    keys = [str(k) for k in np.load(os.path.join(GOLD, "phi3_layer.npz"))["keys"]]    # the reference's fill order
    sd = seeded_fill({k: torch.empty(SHAPES[k]) for k in keys}, 91)           # phi3_layer.npz's weights
    sd = {k: v.requires_grad_() for k, v in sd.items()}
    am = torch.from_numpy(z["attention_mask"])
    cfg = dict(num_attention_heads=2, num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=10000.0,
               sliding_window=int(z["window"]))
    assert not P.sliding_mask(S, S, int(z["window"]), am)[1, S - 1].any()     # the fixture has a row that sees no key
    x = torch.from_numpy(z["x"]).requires_grad_()
    pos = torch.from_numpy(z["pos"])
    out = R.layer(sd, "", cfg, x, pos, am)
    live = am.bool()                                              # the reference's fully masked rows average all keys
    with torch.no_grad():
        assert torch.equal(out[live], P.layer(sd, "", cfg, x, pos, am)[live])   # the oracle's forward, bit for bit
    out.backward(torch.from_numpy(z["dout"]))
    torch.testing.assert_close(out[live], torch.from_numpy(z["out"])[live], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(x.grad, torch.from_numpy(z["dx"]), rtol=1e-4, atol=1e-5)
    for k in SHAPES:
        g = sd[k].grad
        assert torch.isfinite(g).all(), k
        for i, t in enumerate(R.sketch(g)):                       # the fixture keeps sketches of the weight gradients
            want = torch.from_numpy(z[f"grad{i}.{k}"]).double()
            torch.testing.assert_close(t.double(), want, rtol=1e-4, atol=1e-4 * want.abs().max().item(), msg=k)


@needs_no_gpu
def test_tiny_phi3_trains_like_the_oracle_with_the_window_on_every_attention_call(monkeypatch):
    calls = []
    _install(monkeypatch, calls)
    cfg, model = _model()
    ids, am, labels = _batch(cfg.vocab_size)
    assert not P.sliding_mask(S, S, W, am)[1, S - 1].any()
    loss = model(input_ids=ids, attention_mask=am, labels=labels).loss
    loss.backward()
    L = cfg.num_hidden_layers
    assert calls == [("fwd", W)] * L + [("bwd", W)] * L            # both attention calls of every layer, windowed
    want_loss, want = _oracle_loss_and_grads(model, cfg, ids, am, labels)
    assert abs(loss.item() - want_loss) < 2e-2 * want_loss, (loss.item(), want_loss)
    got = _grads(model)
    assert set(got) == set(want)
    for n, g in got.items():
        assert torch.isfinite(g).all(), n
        assert _rel(g, want[n]) < 4e-2, (n, _rel(g, want[n]))       # bf16-rounded stages against fp32


@needs_no_gpu
def test_recompute_on_and_off_give_identical_gradients(monkeypatch):
    calls = []
    _install(monkeypatch, calls)
    cfg, model = _model()
    ids, am, labels = _batch(cfg.vocab_size)
    res = []
    for recompute in (False, True):
        calls.clear()
        model.gradient_checkpointing = recompute
        model.get_model().gradient_checkpointing = recompute
        model.zero_grad(set_to_none=True)
        model(input_ids=ids, attention_mask=am, labels=labels).loss.backward()
        res.append(_grads(model))
        L = cfg.num_hidden_layers
        assert calls.count(("fwd", W)) == (2 * L if recompute else L) and calls.count(("bwd", W)) == L
        assert all(w == W for _, w in calls)
    for n in res[0]:
        assert torch.equal(res[0][n], res[1][n]), n


@needs_no_gpu
def test_fused_leaves_receive_their_gradients_in_autograd_and_in_main_grad(monkeypatch):
    calls = []
    _install(monkeypatch, calls)
    cfg, model = _model()
    ids, am, labels = _batch(cfg.vocab_size)
    model(input_ids=ids, attention_mask=am, labels=labels).loss.backward()
    plain = _grads(model)
    fused = [n for n in plain if n.endswith(("qkv_proj.weight", "gate_up_proj.weight"))]
    assert len(fused) == 2 * cfg.num_hidden_layers
    for n in fused:
        assert plain[n].abs().sum() > 0, n
    model.zero_grad(set_to_none=True)
    from cambrian_b200.engine import TrainEngine
    eng = TrainEngine(model, lr=1e-3, bucket_mb=1.0)
    eng.zero_grad()
    model(input_ids=ids, attention_mask=am, labels=labels).loss.backward()
    for n, p in model.named_parameters():
        assert p.grad is None, n                                  # everything went to main_grad
        assert torch.equal(p.main_grad.float(), plain[n]), n
    eng.step()


def test_cpu_or_fp32_parameters_are_refused():
    cfg, model = tiny_phi3(window=W, layers=1)
    ids = torch.zeros(1, 4, dtype=torch.long)
    for m in (model, model.to(torch.bfloat16)):                   # fp32 on the CPU, then bf16 on the CPU
        with pytest.raises(NotImplementedError, match="Phi3 trains in bf16 on CUDA only.*backward"):
            m(input_ids=ids)
    from cambrian_b200.engine import TrainEngine
    with pytest.raises(NotImplementedError, match="Phi3 trains in bf16 on CUDA only.*backward"):
        TrainEngine(model)


@pytest.mark.parametrize("field", ["attention_dropout", "resid_pdrop", "embd_pdrop"])
def test_dropout_is_refused_in_training(field):
    cfg, model = tiny_phi3(window=W, layers=1)
    setattr(model.config, field, 0.1)
    with pytest.raises(NotImplementedError, match=f"Phi3 with {field}=0.1"):
        model(input_ids=torch.zeros(1, 4, dtype=torch.long))
    from cambrian_b200.engine import TrainEngine
    with pytest.raises(NotImplementedError, match=field):
        TrainEngine(model)


def test_fp8_training_is_refused():
    cfg, model = tiny_phi3(window=W, layers=1)
    model.config.fp8_training = True
    with pytest.raises(NotImplementedError, match="Phi3 with fp8_training"):
        model(input_ids=torch.zeros(1, 4, dtype=torch.long))
    from cambrian_b200.engine import TrainEngine
    with pytest.raises(NotImplementedError, match="fp8_training"):
        TrainEngine(model)
