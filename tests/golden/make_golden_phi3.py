"""Generates the Cambrian-Phi3 golden fixtures from the UNMODIFIED reference (run where the reference tree exists;
nothing else in the repository needs it).

    python tests/golden/make_golden_phi3.py

  phi3_mask.npz    the sliding-window mask the reference's Phi3Model builds, for a short left-padded batch at a small W,
                   and flash-attn's rule (one more key) for contrast
  phi3_layer.npz   the reference's Phi3DecoderLayer (eager attention) on seeded weights (`seeded_fill` of
                   make_golden.py) and inputs under that mask, with its state-dict keys
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from make_golden import seeded_fill  # noqa: E402


PHI3_W = 5   # small sliding window for the Phi-3 fixtures


def phi3_reference_mask(attention_mask, S, W, dtype=torch.float32):
    """The 4-D additive mask the reference's Phi3Model builds (modeling_phi3.py:1180-1186) with
    `_prepare_4d_causal_attention_mask(attention_mask, (B, S), embeds, 0, sliding_window=W)`.  The reference pins
    transformers 4.37.0, whose `_make_causal_mask` masks key slot j from query slot i when i - j >= W
    (`1 - triu(ones, diagonal=past - W + 1)`).  Later releases changed that line to `tril(ones, diagonal=past - W - 1)`,
    masking only i - j >= W + 1 (flash-attn's window_size=(W, W)).  Under such a release the reference's mask is the
    installed function's at sliding_window = W - 1; under 4.37 it is the function's at W."""
    import transformers
    from transformers.modeling_attn_mask_utils import _prepare_4d_causal_attention_mask
    major, minor = (int(x) for x in transformers.__version__.split(".")[:2])
    w_arg = W if (major, minor) < (4, 38) else W - 1
    emb = torch.zeros(attention_mask.shape[0], S, 8, dtype=dtype)
    return _prepare_4d_causal_attention_mask(attention_mask, (attention_mask.shape[0], S), emb, 0, sliding_window=w_arg)


def make_phi3():
    """phi3_mask.npz: the reference's sliding-window mask (additive, fp32) for a left-padded batch of 12 positions at
    W = 5, and the flash-attn rule's for contrast.  phi3_layer.npz: the reference's Phi3DecoderLayer (eager attention)
    on seeded weights and inputs with that mask, for the oracle restatement (oracle/phi3_oracle.py)."""
    from transformers.modeling_attn_mask_utils import _prepare_4d_causal_attention_mask
    from oracle import ref_shim
    S, W = 12, PHI3_W
    am = torch.ones(2, S, dtype=torch.long)
    am[1, :3] = 0                                              # left padding in the second row
    mask = phi3_reference_mask(am, S, W)
    emb = torch.zeros(2, S, 8)
    fa = _prepare_4d_causal_attention_mask(am, (2, S), emb, 0, sliding_window=W)    # i - j <= W (flash-attn's rule)
    np.savez_compressed(os.path.join(HERE, "phi3_mask.npz"), attention_mask=am.numpy(), window=np.int64(W),
                        mask=mask.numpy(), mask_flash=fa.numpy())
    mp = ref_shim.ref_module("cambrian.model.language_model.phi3.modeling_phi3")
    cp = ref_shim.ref_module("cambrian.model.language_model.phi3.configuration_phi3")
    cfg = cp.Phi3Config(vocab_size=64, hidden_size=192, intermediate_size=256, num_hidden_layers=1,
                        num_attention_heads=2, num_key_value_heads=2, sliding_window=W, rope_theta=10000.0,
                        max_position_embeddings=64)
    cfg._attn_implementation = "eager"
    cfg.rope_scaling = None     # newer transformers fill in a default rope dict; the reference reads None as plain RoPE
    lay = mp.Phi3DecoderLayer(cfg, 0).eval()
    lay.load_state_dict(seeded_fill(lay, 91))
    rng = np.random.default_rng(92)
    x = torch.from_numpy(rng.standard_normal((2, S, 192)).astype(np.float32))
    pos = (am.cumsum(1) - 1).clamp(min=0)
    with torch.no_grad():
        out = lay(x, attention_mask=mask, position_ids=pos)[0]
    np.savez_compressed(os.path.join(HERE, "phi3_layer.npz"), x=x.numpy(), pos=pos.numpy(), out=out.numpy(),
                        keys=np.array(list(lay.state_dict().keys())))
    print("phi3 fixtures written", tuple(out.shape))


if __name__ == "__main__":
    make_phi3()
