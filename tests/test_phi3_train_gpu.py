"""Cambrian-Phi3 training on the GPU: the head-dim-96 and sliding-window flash-attention backward against an fp64
autograd reference of the pinned mask (oracle/phi3_oracle.py: 0 <= i - j < W in cache slots) with an eager-bf16 arm,
a Phi-3-mini-shaped decoder layer against the fp32 oracle's differentiable restatement (tests/phi3_train_reference.py),
and a tiny Phi-3 under autograd and TrainEngine."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import ParityCollector, oracle_device  # noqa: E402
from test_phi3_gpu import tiny_phi3  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"


def _inputs(B, Sq, Skv, nh, nkv, hd, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    q = torch.randn(B, Sq, nh, hd, device=dev, generator=g).bfloat16()
    k = torch.randn(B, Skv, nkv, hd, device=dev, generator=g).bfloat16()
    v = torch.randn(B, Skv, nkv, hd, device=dev, generator=g).bfloat16()
    do = torch.randn(B, Sq, nh, hd, device=dev, generator=g).bfloat16()
    return q, k, v, do


def _ref_grads(q, k, v, do, window, kmask, dtype):
    """dq, dk, dv of softmax attention under the pinned rule, by autograd in `dtype` (fp64: the reference; bf16: the
    reference's eager numerics, softmax in fp32).  A query row that sees no key has zero output and zero gradients."""
    from oracle.phi3_oracle import sliding_mask
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    Q, K, V = (t.to(dtype).detach().requires_grad_() for t in (q, k, v))
    Kr = K.transpose(1, 2).repeat_interleave(nh // nkv, 1)
    Vr = V.transpose(1, 2).repeat_interleave(nh // nkv, 1)
    s = (Q.transpose(1, 2) @ Kr.transpose(-1, -2)) * hd ** -0.5
    allow = sliding_mask(Sq, Skv, window, None if kmask is None else kmask.cpu()).to(q.device)[:, None]
    live = allow.any(-1, keepdim=True)
    sf = s.to(torch.float64 if dtype == torch.float64 else torch.float32)
    p = torch.softmax(sf.masked_fill(~allow, float("-inf")).masked_fill(~live, 0.0), -1).masked_fill(~live, 0.0)
    o = (p.to(dtype) @ Vr).transpose(1, 2)
    return [g.double() for g in torch.autograd.grad(o, [Q, K, V], do.to(dtype))]


def _kernel(q, k, v, do, window, kmask):
    from cambrian_b200 import ops
    win = {"window": window} if window else {}
    o, lse = ops.attn_fwd(q, k, v, causal=True, kmask=kmask, need_lse=True, **win)
    return ops.attn_bwd(q, k, v, o, do, lse, causal=True, kmask=kmask, **win)


def _check(q, k, v, do, window, kmask, what, pc):
    got = _kernel(q, k, v, do, window, kmask)
    ref = _ref_grads(q, k, v, do, window, kmask, torch.float64)
    eager = _ref_grads(q, k, v, do, window, kmask, torch.bfloat16)
    for name, g, r, e in zip(("dq", "dk", "dv"), got, ref, eager):
        assert torch.isfinite(g.float()).all(), f"{what} {name}: non-finite"
        if window == 1 and name != "dv":
            # every query sees only itself: P = 1 and dS = P (dP - delta) = 0, so dq and dk are exactly zero and a
            # relative error is undefined; the kernel's dP and delta differ only by fp32 summation order
            assert r.abs().max() < 1e-9 and g.abs().max() < 1e-4, f"{what} {name}: max {g.abs().max().item():.3e}"
            continue
        pc.check(g.double(), r, e, f"{what} {name}")
    return got


def _kmask(B, S, pad):
    if pad == "none":
        return None
    km = torch.ones(B, S, dtype=torch.bool, device=dev)
    if pad == "left":
        km[1, :37] = False
    else:
        km[1, S - S // 2:] = False                     # right padding longer than W for every W below S // 2
    return km


@pytest.mark.parametrize("S,window", [(300, 301), (300, 300), (300, 299), (300, 100), (300, 1), (1000, 257)])
@pytest.mark.parametrize("pad", ["none", "left", "right"])
@pytest.mark.parametrize("nh,nkv", [(4, 4), (4, 2)])
def test_attn_bwd_hd96_window_matches_fp64(S, window, pad, nh, nkv):
    pc = ParityCollector()
    q, k, v, do = _inputs(2, S, S, nh, nkv, 96, seed=S + window + nkv)
    _check(q, k, v, do, window, _kmask(2, S, pad), f"hd96 S={S} W={window} pad={pad} nh={nh} nkv={nkv}", pc)
    pc.done()


def test_attn_bwd_hd96_window_sq_below_skv_and_4096():
    """Queries at the end of a longer key range (Sq < Skv), and S = 4096 at Phi-3's W = 2047."""
    pc = ParityCollector()
    q, k, v, do = _inputs(2, 130, 900, 4, 2, 96, seed=130)
    _check(q, k, v, do, 128, None, "hd96 Sq=130 Skv=900 W=128", pc)
    q, k, v, do = _inputs(1, 4096, 4096, 2, 2, 96, seed=4096)
    _check(q, k, v, do, 2047, None, "hd96 S=4096 W=2047", pc)
    pc.done()


def test_fully_masked_rows_get_zero_dq_and_everything_is_finite():
    """Right padding longer than W: the last padded queries see no key (lse = +inf).  dO on those rows is random."""
    S, W = 333, 40
    q, k, v, do = _inputs(2, S, S, 4, 2, 96, seed=7)
    km = torch.ones(2, S, dtype=torch.bool, device=dev)
    km[1, 200:] = False                                          # slots 240.. of row 1 see no key
    dq, dk, dv = _kernel(q, k, v, do, W, km)
    for t in (dq, dk, dv):
        assert torch.isfinite(t.float()).all()
    assert torch.count_nonzero(dq[1, 240:]) == 0
    assert torch.count_nonzero(dq[1, :239]) > 0
    assert torch.count_nonzero(dk[1, 200:]) == 0 and torch.count_nonzero(dv[1, 200:]) == 0   # padded keys


@pytest.mark.parametrize("hd,nh,nkv", [(64, 6, 6), (128, 8, 2)])
def test_attn_bwd_window_hd64_hd128_match_fp64(hd, nh, nkv):
    pc = ParityCollector()
    q, k, v, do = _inputs(2, 520, 520, nh, nkv, hd, seed=hd)
    _check(q, k, v, do, 150, _kmask(2, 520, "right"), f"hd{hd} S=520 W=150", pc)
    pc.done()


def test_attn_bwd_hd96_without_window_matches_fp64():
    pc = ParityCollector()
    q, k, v, do = _inputs(2, 700, 700, 4, 2, 96, seed=700)
    _check(q, k, v, do, 0, _kmask(2, 700, "left"), "hd96 S=700 no window", pc)
    pc.done()


def _bwd_window_abi(q, k, v, o, do, lse, window):
    """cb_attn_bwd_window called directly (window = 0 included, which ops.attn_bwd routes to cb_attn_bwd)."""
    from cambrian_b200 import _lib
    from cambrian_b200.ops import _bshd_strides, ptr, stream
    B, S, nh, hd = q.shape
    nkv = k.shape[2]
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    delta = torch.empty(B, nh, S, dtype=torch.float32, device=dev)
    st = [x for t in (q, k, v, o, do, dq, dk, dv) for x in _bshd_strides(t, hd)]
    rc = _lib.load().cb_attn_bwd_window(ptr(q), ptr(k), ptr(v), ptr(o), ptr(do), ptr(lse), ptr(delta), ptr(dq),
                                        ptr(dk), ptr(dv), None, B, nh, nkv, S, S, hd, *st, hd ** -0.5, 1, window,
                                        stream())
    assert rc == 0
    return dq, dk, dv


@pytest.mark.parametrize("hd,nh,nkv", [(64, 6, 6), (96, 4, 4), (128, 8, 2)])
def test_window_zero_and_unreachable_window_are_the_plain_kernels_bitwise(hd, nh, nkv):
    from cambrian_b200 import ops
    S = 333
    q, k, v, do = _inputs(2, S, S, nh, nkv, hd, seed=hd + 1)
    o, lse = ops.attn_fwd(q, k, v, causal=True, need_lse=True)
    base = ops.attn_bwd(q, k, v, o, do, lse, causal=True)
    for got in (_bwd_window_abi(q, k, v, o, do, lse, 0), ops.attn_bwd(q, k, v, o, do, lse, causal=True, window=S),
                ops.attn_bwd(q, k, v, o, do, lse, causal=True, window=10 * S)):
        for a, b in zip(base, got):
            assert torch.equal(a, b)
    hidden = ops.attn_bwd(q, k, v, o, do, lse, causal=True, window=64)
    assert not torch.equal(base[0], hidden[0]) and not torch.equal(base[1], hidden[1])
    again = ops.attn_bwd(q, k, v, o, do, lse, causal=True, window=64)            # bit-reproducible: no atomics
    for a, b in zip(hidden, again):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------- the layer
def _phi3_layer(H, nh, I, W, seed):
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3Config, CBPhi3DecoderLayer
    cfg = CambrianPhi3Config(hidden_size=H, num_attention_heads=nh, intermediate_size=I, num_hidden_layers=1,
                             sliding_window=W, max_position_embeddings=4096)
    torch.manual_seed(seed)
    lay = CBPhi3DecoderLayer(cfg, 0)
    with torch.no_grad():
        for n, p in lay.named_parameters():
            if n.endswith("layernorm.weight"):
                p.uniform_(0.5, 1.5)
            else:
                p.normal_(0, H ** -0.5)
    return cfg, lay.to(dev, torch.bfloat16)


def _run_layer(lay, cfg, x, km, recompute):
    from cambrian_b200.model.language_model.cambrian_llama import rope_tables
    B, S, H = x.shape
    cos, sin = rope_tables(cfg, dev)
    rt = dict(pos=torch.arange(S, device=dev).repeat(B), cos=cos, sin=sin, kmask=km, hf_cast=False,
              recompute=recompute)
    xx = x.detach().clone().requires_grad_()
    lay.zero_grad(set_to_none=True)
    out = lay(xx, rt)
    return out, xx


def test_phi3_mini_layer_at_4096_matches_the_fp32_oracle():
    """Hidden 3072 / 32 heads (hd 96) / 8192, S = 4096, W = 2047, right padding longer than W in the second row; the
    upstream gradient is zero on padded rows, as the loss's ignored labels make it."""
    import phi3_train_reference as P
    H, nh, I, S, W = 3072, 32, 8192, 4096, 2047
    cfg, lay = _phi3_layer(H, nh, I, W, seed=3)
    g = torch.Generator(device=dev).manual_seed(4)
    x = torch.randn(2, S, H, device=dev, generator=g).bfloat16()
    km = torch.ones(2, S, dtype=torch.bool, device=dev)
    km[1, 1500:] = False
    dout = (torch.randn(2, S, H, device=dev, generator=g) * km[..., None]).bfloat16()
    res = {}
    for recompute in (False, True):
        out, xx = _run_layer(lay, cfg, x, km, recompute)
        out.backward(dout)
        res[recompute] = [out.detach(), xx.grad] + [p.grad.clone() for _, p in lay.named_parameters()]
    for a, b in zip(res[False], res[True]):
        assert torch.equal(a, b)                                  # recompute changes nothing, bit for bit
    names = ["out", "dx"] + [n for n, _ in lay.named_parameters()]
    sd32 = {n: p.detach().float() for n, p in lay.state_dict().items()}
    arms = []
    odev = oracle_device()
    for dt in (torch.float32, torch.bfloat16):
        sd = {n: t.detach().to(odev, dt).requires_grad_() for n, t in sd32.items()}
        xo = x.detach().to(odev, dt).requires_grad_()
        ocfg = dict(num_attention_heads=nh, num_key_value_heads=nh, rms_norm_eps=cfg.rms_norm_eps,
                    rope_theta=cfg.rope_theta, sliding_window=W)
        pos = torch.arange(S, device=odev)[None].expand(2, S)
        out = P.layer(sd, "", ocfg, xo, pos, km.to(odev))
        out.backward(dout.to(odev, dt))
        arms.append([out.detach(), xo.grad] + [sd[n].grad for n, _ in lay.named_parameters()])
        del sd, xo, out
    live = km.bool()
    pc = ParityCollector()
    for i, n in enumerate(names):
        got, r32, eag = res[False][i], arms[0][i], arms[1][i]
        if n == "out":                                            # padded rows are never read
            got, r32, eag = got[live], r32[live], eag[live]
        assert torch.isfinite(got.float()).all(), n
        pc.check(got.double(), r32.double(), eag.double(), f"phi3-mini layer S=4096 W=2047 {n}")
    pc.done()


# ---------------------------------------------------------------------------------------------------------- the model
def _batch(vocab, B=2, S=48, valid=30, seed=21):
    ids = torch.randint(3, vocab, (B, S), generator=torch.Generator().manual_seed(seed))
    am = torch.ones(B, S, dtype=torch.long)
    am[1, valid:] = 0
    return ids.to(dev), am.to(dev), ids.masked_fill(am == 0, -100).to(dev)


def _tame(model):
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith("o_proj.weight"):
                p.div_(15.0)
    return model


def test_tiny_phi3_loss_and_gradients_match_the_fp32_oracle():
    import phi3_train_reference as P
    W = 8
    cfg, model = tiny_phi3(window=W, layers=2)
    model = _tame(model).to(dev, torch.bfloat16).train()
    ids, am, labels = _batch(cfg.vocab_size)
    loss = model(input_ids=ids, attention_mask=am, labels=labels).loss
    loss.backward()
    ocfg = dict(num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads,
                num_hidden_layers=cfg.num_hidden_layers, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
                sliding_window=W)
    arms = []
    for dt in (torch.float32, torch.bfloat16):
        sd = {k: v.detach().to(dt).requires_grad_() for k, v in model.state_dict().items()}
        lg = P.logits(sd, ocfg, ids, kmask=am).float()
        ref_loss = torch.nn.functional.cross_entropy(lg[:, :-1].reshape(-1, lg.shape[-1]), labels[:, 1:].reshape(-1),
                                                     ignore_index=-100)
        ref_loss.backward()
        arms.append((ref_loss.item(), {k: v.grad for k, v in sd.items()}))
    assert abs(loss.item() - arms[0][0]) <= 3 * max(abs(arms[1][0] - arms[0][0]), 1e-3 * arms[0][0]), \
        (loss.item(), arms[0][0], arms[1][0])
    pc = ParityCollector()
    for n, p in model.named_parameters():
        assert torch.isfinite(p.grad.float()).all(), n
        pc.check(p.grad.double(), arms[0][1][n].double(), arms[1][1][n].double(), f"tiny phi3 grad {n}")
    pc.done()


def _engine_run(steps, W=8, seed=5, lr=2e-3):
    from cambrian_b200.engine import TrainEngine
    cfg, model = tiny_phi3(window=W, layers=2, seed=seed)
    model = _tame(model).to(dev, torch.bfloat16).train()
    model.gradient_checkpointing = model.get_model().gradient_checkpointing = True
    ids, am, labels = _batch(cfg.vocab_size)
    eng = TrainEngine(model, lr=lr)
    losses = []
    for _ in range(steps):
        eng.zero_grad()
        loss = model(input_ids=ids, attention_mask=am, labels=labels).loss
        loss.backward()
        eng.step()
        losses.append(loss.item())
    torch.cuda.synchronize()
    return losses, eng.flat_p.clone()


def test_three_train_engine_steps_are_bitwise_reproducible():
    l1, p1 = _engine_run(3)
    l2, p2 = _engine_run(3)
    assert l1 == l2 and torch.equal(p1, p2), (l1, l2)


def test_memorisation_run_drives_the_loss_down():
    losses, _ = _engine_run(100, lr=3e-3)
    print(f"phi3 memorisation: initial loss {losses[0]:.4f}, final loss {losses[-1]:.3e}")
    assert all(torch.isfinite(torch.tensor(losses)))
    assert losses[-1] < 0.1 * losses[0], (losses[0], losses[-1])


# ---------------------------------------------------------------------------------------------- multimodal plumbing
def _phi3_from_llama(llama, cfg):
    """CambrianPhi3ForCausalLM with the LLaMA model's configuration (towers, SVA connector, in-LLM SVA sites) and
    weights: qkv_proj = cat(q, k, v), gate_up_proj = cat(gate, up), everything else as it is; no window."""
    import test_modules_gpu as T
    from helpers import rope_theta
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3Config, CambrianPhi3ForCausalLM
    d = {k: v for k, v in cfg.to_dict().items() if k not in ("model_type", "architectures", "rope_scaling",
                                                              "rope_parameters", "transformers_version")}
    pcfg = CambrianPhi3Config(**d)
    pcfg.rope_theta, pcfg.sliding_window = rope_theta(cfg), None
    torch.manual_seed(3)
    phi = CambrianPhi3ForCausalLM(pcfg)
    for t in phi.get_model().vision_tower_aux_list:
        t.load_model()
    phi = T._cuda_bf16(phi)
    for tl, tp in zip(llama.get_model().vision_tower_aux_list, phi.get_model().vision_tower_aux_list):
        tp.to(device=dev, dtype=torch.bfloat16)
        tp.load_state_dict(tl.state_dict())
    sd, mapped = llama.state_dict(), {}
    for k, v in sd.items():
        if k.endswith("self_attn.q_proj.weight"):
            pre = k[: -len("q_proj.weight")]
            mapped[pre + "qkv_proj.weight"] = torch.cat([v, sd[pre + "k_proj.weight"], sd[pre + "v_proj.weight"]])
        elif k.endswith("mlp.gate_proj.weight"):
            pre = k[: -len("gate_proj.weight")]
            mapped[pre + "gate_up_proj.weight"] = torch.cat([v, sd[pre + "up_proj.weight"]])
        elif not (k.startswith("model.layers.") and
                  k.endswith(("self_attn.k_proj.weight", "self_attn.v_proj.weight", "mlp.up_proj.weight"))):
            mapped[k] = v
    missing, unexpected = phi.load_state_dict(mapped, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return phi


def _mm_step(model, eng, batch):
    ids, labels, attn, pos, images, masks = batch
    eng.zero_grad()
    loss = model(input_ids=ids.to(dev), labels=labels.to(dev), attention_mask=attn.to(dev), position_ids=pos.to(dev),
                 images=[i.to(dev).bfloat16() for i in images],
                 image_aux_attention_masks_list=[m.to(dev) for m in masks]).loss
    loss.backward()
    eng.step()
    torch.cuda.synchronize()
    return loss.detach().clone()


def test_multimodal_phi3_trains_exactly_like_llama_with_mapped_weights():
    import test_modules_gpu as T
    from helpers import tiny_cambrian_config
    cfg = tiny_cambrian_config()
    llama = T._build_tiny_model(cfg).train()
    phi = _phi3_from_llama(llama, cfg).train()
    from cambrian_b200.engine import TrainEngine
    batch = T._tiny_batch(cfg)
    e_llama, e_phi = TrainEngine(llama, lr=1e-3, max_grad_norm=None), TrainEngine(phi, lr=1e-3, max_grad_norm=None)
    l_llama, l_phi = _mm_step(llama, e_llama, batch), _mm_step(phi, e_phi, batch)
    assert torch.equal(l_llama, l_phi), (l_llama.item(), l_phi.item())
    sd_l, sd_p = llama.state_dict(), phi.state_dict()
    for k, v in sd_p.items():
        if k.endswith("qkv_proj.weight"):
            pre = k[: -len("qkv_proj.weight")]
            want = torch.cat([sd_l[pre + "q_proj.weight"], sd_l[pre + "k_proj.weight"], sd_l[pre + "v_proj.weight"]])
        elif k.endswith("gate_up_proj.weight"):
            pre = k[: -len("gate_up_proj.weight")]
            want = torch.cat([sd_l[pre + "gate_proj.weight"], sd_l[pre + "up_proj.weight"]])
        else:
            want = sd_l[k]
        assert torch.equal(v, want), k                              # the same updated weights, bit for bit
    for layer in phi.get_model().layers:                            # now a window shorter than the sequence
        layer.window = 16
    assert not torch.equal(_mm_step(llama, e_llama, batch), _mm_step(phi, e_phi, batch))
