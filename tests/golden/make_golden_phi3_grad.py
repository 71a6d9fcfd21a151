"""Generates the Cambrian-Phi3 gradient fixture from the UNMODIFIED reference (run where the reference tree exists;
nothing else in the repository needs it).

    python tests/golden/make_golden_phi3_grad.py

  phi3_layer_grad.npz
      the reference's Phi3DecoderLayer in train mode (eager attention, dropouts 0) with phi3_layer.npz's seeded weights
      (`seeded_fill(layer, 91)`), on a right-padded batch of 12 positions with 7 valid tokens in the second row: at
      W = 5 its query slots 11.. see no key.  Records x, the upstream gradient (seeded, zero on padded rows, as the
      loss's ignored labels make it), the output, dx, the two RMSNorm weight gradients in full, and of each projection
      weight gradient the two-sided random sketch of tests/phi3_train_reference.py (`sketch`) — the full matrices
      would make the fixture a megabyte.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from make_golden import seeded_fill  # noqa: E402
from make_golden_phi3 import PHI3_W, phi3_reference_mask  # noqa: E402
from phi3_train_reference import sketch  # noqa: E402

S, VALID = 12, 7


def make_phi3_grad():
    from oracle import ref_shim
    am = torch.ones(2, S, dtype=torch.long)
    am[1, VALID:] = 0
    mask = phi3_reference_mask(am, S, PHI3_W)
    mp = ref_shim.ref_module("cambrian.model.language_model.phi3.modeling_phi3")
    cp = ref_shim.ref_module("cambrian.model.language_model.phi3.configuration_phi3")
    cfg = cp.Phi3Config(vocab_size=64, hidden_size=192, intermediate_size=256, num_hidden_layers=1,
                        num_attention_heads=2, num_key_value_heads=2, sliding_window=PHI3_W, rope_theta=10000.0,
                        max_position_embeddings=64, attention_dropout=0.0, resid_pdrop=0.0, embd_pdrop=0.0)
    cfg._attn_implementation = "eager"
    cfg.rope_scaling = None     # newer transformers fill in a default rope dict; the reference reads None as plain RoPE
    lay = mp.Phi3DecoderLayer(cfg, 0).train()
    lay.load_state_dict(seeded_fill(lay, 91))
    rng = np.random.default_rng(93)
    x = torch.from_numpy(rng.standard_normal((2, S, 192)).astype(np.float32)).requires_grad_(True)
    dout = torch.from_numpy(rng.standard_normal((2, S, 192)).astype(np.float32)) * am[..., None].float()
    pos = torch.arange(S)[None].expand(2, S)
    out = lay(x, attention_mask=mask, position_ids=pos)[0]
    out.backward(dout)
    grads = {}
    for k, p in lay.named_parameters():
        for i, t in enumerate(sketch(p.grad)):
            grads[f"grad{i}.{k}"] = t.numpy().astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "phi3_layer_grad.npz"), x=x.detach().numpy(), pos=pos.numpy(),
                        attention_mask=am.numpy(), window=np.int64(PHI3_W), dout=dout.numpy(),
                        out=out.detach().numpy(), dx=x.grad.numpy(), **grads)
    print("phi3 gradient fixture written", sorted(grads))


if __name__ == "__main__":
    make_phi3_grad()
