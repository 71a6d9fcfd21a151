"""Cambrian-Phi3 on the GPU: the head-dim-96 and sliding-window flash-attention forward against an fp64 reference of
the reference's mask rule (oracle/phi3_oracle.py: 0 <= i - j < W in cache slots), and greedy generation of a tiny
random Phi-3-shaped model past W generated positions, token-exact against the fp32 oracle, graph and eager loops alike."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import assert_parity  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"


def _qkv(B, Sq, Skv, nh, nkv, hd, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    q = torch.randn(B, Sq, nh, hd, device=dev, generator=g).bfloat16()
    k = torch.randn(B, Skv, nkv, hd, device=dev, generator=g).bfloat16()
    v = torch.randn(B, Skv, nkv, hd, device=dev, generator=g).bfloat16()
    return q, k, v


def _ref(q, k, v, window, kmask, dtype):
    """Softmax attention under the pinned rule in `dtype` (fp64: the reference; bf16: the reference's eager numerics)."""
    from oracle.phi3_oracle import sliding_mask
    B, Sq, nh, hd = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    Q = q.to(dtype).transpose(1, 2)
    K = k.to(dtype).transpose(1, 2).repeat_interleave(nh // nkv, 1)
    V = v.to(dtype).transpose(1, 2).repeat_interleave(nh // nkv, 1)
    s = (Q @ K.transpose(-1, -2)).float() * hd ** -0.5
    allow = sliding_mask(Sq, Skv, window, None if kmask is None else kmask.cpu()).to(q.device)[:, None]
    p = torch.softmax(s.double().masked_fill(~allow, float("-inf")), -1).nan_to_num(0.0)
    return (p.to(dtype) @ V).transpose(1, 2).double()


@pytest.mark.parametrize("S,window", [(300, 301), (300, 300), (300, 299), (300, 100), (300, 1), (1000, 257)])
@pytest.mark.parametrize("padded", [False, True])
def test_attn_hd96_window_matches_fp64(S, window, padded):
    from cambrian_b200 import ops
    B, nh, hd = 2, 4, 96
    q, k, v = _qkv(B, S, S, nh, nh, hd, seed=S + window)
    kmask = None
    if padded:
        kmask = torch.ones(B, S, dtype=torch.bool, device=dev)
        kmask[1, :37] = False                                   # left padding: slots, not positions, count
    got = ops.attn_fwd(q, k, v, causal=True, kmask=kmask, window=window)
    ref = _ref(q, k, v, window, kmask, torch.float64)
    eager = _ref(q, k, v, window, kmask, torch.bfloat16)
    rows = slice(None) if not padded else slice(37, None)      # fully padded query rows are never read
    assert_parity(got[1:, rows].double(), ref[1:, rows], eager[1:, rows], f"hd96 S={S} W={window} padded={padded}")
    assert_parity(got[:1].double(), ref[:1], eager[:1], f"hd96 S={S} W={window} row0")


def test_attn_window_decode_shapes_match_fp64():
    """Queries at the end of a longer key range (a prefilled cache: Sq < Skv), as the eager decode loop calls it."""
    from cambrian_b200 import ops
    for Sq, Skv, W in ((1, 700, 256), (5, 700, 256), (130, 900, 128)):
        q, k, v = _qkv(2, Sq, Skv, 4, 4, 96, seed=Skv + Sq)
        got = ops.attn_fwd(q, k, v, causal=True, window=W)
        assert_parity(got.double(), _ref(q, k, v, W, None, torch.float64), _ref(q, k, v, W, None, torch.bfloat16),
                      f"decode Sq={Sq} Skv={Skv} W={W}")


def test_window_zero_is_the_plain_kernel_bitwise():
    """window = 0 through the new entry point, and a window no query can reach, are the plain kernel bit for bit
    (hd 64 and 128 included); a window that hides keys changes the result."""
    from cambrian_b200 import ops
    for hd, nh, nkv in ((64, 6, 6), (96, 4, 4), (128, 8, 2)):
        q, k, v = _qkv(2, 333, 333, nh, nkv, hd, seed=hd)
        base = ops.attn_fwd(q, k, v, causal=True)
        assert torch.equal(base, ops.attn_fwd(q, k, v, causal=True, window=333))
        from cambrian_b200 import _lib
        from cambrian_b200.ops import _bshd_strides, ptr, stream
        o = torch.empty_like(base)
        st = [x for t in (q, k, v, o) for x in _bshd_strides(t, hd)]
        rc = _lib.load().cb_attn_fwd_window(ptr(q), ptr(k), ptr(v), ptr(o), None, None, 2, nh, nkv, 333, 333, hd, *st,
                                            hd ** -0.5, 1, 0, stream())
        assert rc == 0
        assert torch.equal(base, o)
        assert not torch.equal(base, ops.attn_fwd(q, k, v, causal=True, window=64))


def test_window_4096_skips_tiles_and_matches_fp64():
    """S = 4096 at Phi-3's W = 2047: most key tiles of late query tiles are skipped."""
    from cambrian_b200 import ops
    q, k, v = _qkv(1, 4096, 4096, 2, 2, 96, seed=4096)
    got = ops.attn_fwd(q, k, v, causal=True, window=2047)
    assert_parity(got.double(), _ref(q, k, v, 2047, None, torch.float64), _ref(q, k, v, 2047, None, torch.bfloat16),
                  "hd96 S=4096 W=2047")


def tiny_phi3(window=24, layers=3, seed=5):
    from cambrian_b200.model.language_model.cambrian_phi3 import CambrianPhi3Config, CambrianPhi3ForCausalLM
    cfg = CambrianPhi3Config(vocab_size=512, hidden_size=192, intermediate_size=384, num_hidden_layers=layers,
                             num_attention_heads=2, num_key_value_heads=2, max_position_embeddings=256,
                             sliding_window=window, pad_token_id=0, eos_token_id=1, bos_token_id=2)
    torch.manual_seed(seed)
    model = CambrianPhi3ForCausalLM(cfg)
    with torch.no_grad():
        emb = model.get_model().embed_tokens.weight
        emb.normal_(0, 1.0)
        perm = torch.randperm(emb.shape[0], generator=torch.Generator().manual_seed(9))
        model.lm_head.weight.copy_(emb[perm] * 2.0)            # next token = a fixed permutation of the context's mix
        for n_, p in model.named_parameters():                 # a strong attention branch, so that the window changes
            if n_.endswith("o_proj.weight"):                   # the tokens; min fp32 top-1 margin 1.5 at W = 24
                p.mul_(15.0)                                   # (calibrated on the CPU oracle)
            elif n_.endswith("qkv_proj.weight"):
                p.mul_(3.0)
    return cfg, model.eval()


def test_greedy_generate_past_the_window_matches_fp32_oracle():
    from oracle import phi3_oracle as P
    cfg, model = tiny_phi3()
    model = model.to(dev, torch.bfloat16)
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}      # the oracle sees the bf16 weights
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(3, cfg.vocab_size, (2, 40), generator=g)
    am = torch.ones_like(ids)
    am[1, :9] = 0                                               # left padding in the second row
    n_new = 40                                                  # prompt 40 > W = 24, and 40 generated positions
    kw = dict(attention_mask=am.to(dev), max_new_tokens=n_new, do_sample=False, eos_token_id=None)
    graphed = model.generate(ids.to(dev), **kw)
    model.config.disable_decode_graph = True
    eager = model.generate(ids.to(dev), **kw)
    model.config.disable_decode_graph = False
    assert torch.equal(graphed, eager), (graphed.tolist(), eager.tolist())
    ocfg = dict(num_attention_heads=2, num_key_value_heads=2, num_hidden_layers=cfg.num_hidden_layers,
                rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, sliding_window=cfg.sliding_window)
    want, margins = P.greedy(sd, ocfg, ids, n_new, attention_mask=am)
    got = graphed.cpu().tolist()
    assert got == want, (got, want, margins)
    assert len(set(got[0])) >= 8, f"degenerate decode: {got[0]}"
    assert min(margins) > 1.0, f"test model lost its margin (min {min(margins)}): re-calibrate"
    # the window matters here: without it the oracle decodes differently
    nowin, _ = P.greedy(sd, dict(ocfg, sliding_window=None), ids, n_new, attention_mask=am)
    assert nowin != want
