"""Minimal end-to-end use of the drop-in modules on one H100 (random-init, synthetic batch; mirrors what
tests/test_modules_gpu.py exercises — the model / collator / engine calls are the ones a training loop makes).

    python -m cambrian_b200.build          # once
    python examples/train_and_generate.py  # needs cuda:0

Swap `tiny_config()` for a released checkpoint with
`cambrian_b200.checkpoint.load_pretrained_model("nyu-visionx/cambrian-8b")` (same state-dict keys as the reference).
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cambrian_b200.engine import TrainEngine  # noqa: E402
from cambrian_b200.model.language_model.cambrian_llama import CambrianConfig, CambrianLlamaForCausalLM  # noqa: E402
from cambrian_b200.train.collator import valid_label_ranges  # noqa: E402


def tiny_config():
    cfg = CambrianConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=4, num_attention_heads=4,
                         num_key_value_heads=2, vocab_size=1024, max_position_embeddings=512, rope_theta=500000.0)
    q = 4                                                    # 4 x 4 = 16 visual tokens (the 8B model uses 24 x 24)
    cfg.image_token_len = q * q
    cfg.mm_vision_tower_aux_list = ["siglip/CLIP-ViT-SO400M-14-384", "openai/clip-vit-large-patch14-336",
                                    "facebook/dinov2-large-res56", "clip-convnext-XXL-multi-stage-res128"]
    cfg.mm_vision_tower_aux_token_len_list = [q * q, q * q, q * q, (2 * q) ** 2]
    cfg.siglip_config_overrides = dict(hidden_size=288, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                                       image_size=56)
    cfg.clip_config_overrides = dict(hidden_size=256, intermediate_size=512, num_hidden_layers=3, num_attention_heads=4,
                                     image_size=56)
    cfg.dino_config_overrides = dict(hidden_size=384, num_hidden_layers=2, num_attention_heads=6, mlp_ratio=4)
    cfg.convnext_config_overrides = dict(depths=(1, 1, 2, 1), dims=(64, 128, 256, 512), image_size=128)
    cfg.mm_projector_type, cfg.vision_hidden_size = "sva", 1024
    cfg.num_query_group, cfg.query_num_list, cfg.connector_depth, cfg.connector_only = 1, [q * q], 2, False
    cfg.num_of_vision_sampler_layers, cfg.start_of_vision_sampler_layers, cfg.stride_of_vision_sampler_layers = 2, 0, 2
    cfg.image_position, cfg.fused_lm_loss = 5, True
    return cfg


def main():
    dev = torch.device("cuda", 0)
    cfg = tiny_config()
    torch.manual_seed(0)
    model = CambrianLlamaForCausalLM(cfg)
    for tower in model.get_model().vision_tower_aux_list:
        tower.load_model()                                   # random init here; pass state_dict=... for real weights
    model.to(device=dev, dtype=torch.bfloat16).train()
    for tower in model.get_model().vision_tower_aux_list:     # the towers live in a plain list, as in the reference
        tower.to(device=dev, dtype=torch.bfloat16)
    engine = TrainEngine(model, lr=1e-3)                     # flat bf16 params/grads, fp32 master + Adam, fused AdamW

    B, S, q = 2, 96, 4
    span = q * (q + 1)                                       # 16 image tokens + 4 newline tokens
    ids = torch.randint(3, cfg.vocab_size, (B, S))
    ids[:, cfg.image_position] = -200                        # <image> indicator, already expanded as the collator does
    ids[:, cfg.image_position + 1:cfg.image_position + span] = 0
    labels = ids.clone()
    labels[:, :cfg.image_position + span] = -100
    ranges, n_valid = valid_label_ranges(labels)             # host-side hints for the fused lm_head + loss
    images = [torch.randn(B, 3, r, r).bfloat16().to(dev) for r in (56, 56, 56, 128)]
    batch = dict(input_ids=ids.to(dev), labels=labels.to(dev), attention_mask=torch.ones(B, S, dtype=torch.bool, device=dev),
                 position_ids=torch.arange(S, device=dev)[None].expand(B, S).contiguous(), images=images)
    for step in range(5):
        engine.zero_grad()
        out = model(**batch, num_valid_labels=n_valid, label_ranges=ranges, image_positions=[cfg.image_position] * B)
        out.loss.backward()
        engine.step()
        print(f"step {step}: loss {float(out.loss):.4f}")

    model.eval()
    prompt = torch.randint(3, cfg.vocab_size, (1, 12))
    prompt[0, cfg.image_position] = -200                     # bare indicator: generate() expands it
    toks = model.generate(prompt.to(dev), images=[i[:1] for i in images], image_sizes=[(640, 480)], max_new_tokens=8)
    print("generated ids:", toks[0].tolist())


if __name__ == "__main__":
    main()
