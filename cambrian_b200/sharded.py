"""ZeRO-3 style parameter sharding for inference (BASELINE config 5: Cambrian-34B `generate` on 8 GPUs).

The reference reaches this configuration through DeepSpeed ZeRO-3 (`scripts/zero3.json:16-27`) / `device_map="auto"`
(model/builder.py:29-33).  Design (SURVEY.md §8e): one process per GPU, the decoder layers — 97 % of the
parameters — are flattened per layer and every rank keeps 1/world of each layer; a layer's full weights exist only in
one of two staging buffers, all-gathered over NCCL/NVLink one layer AHEAD of the layer being computed, so the gather of
layer i+1 overlaps the GEMMs of layer i.  The gather wraps around (the last layer prefetches layer 0), which keeps the
pipeline full across decode steps.  Embedding, lm_head, final norm, SVA / projector / tower weights stay replicated
(3 % of a 34B model).  The batch is split across ranks; KV caches are local.

Per-GPU footprint for Yi-34B: 60 layers x 1.1 GB / 8 = 8.3 GB of shards + 2 x 1.1 GB staging + ~1.9 GB replicated.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def _round8(n: int) -> int:
    return (n + 7) // 8 * 8


class Zero3Inference:
    LAYER_PARAMS = ("input_layernorm.weight", "self_attn.q_proj.weight", "self_attn.k_proj.weight",
                    "self_attn.v_proj.weight", "self_attn.o_proj.weight", "post_attention_layernorm.weight",
                    "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight")

    def __init__(self, model, process_group=None):
        """`model`: a CambrianLlamaForCausalLM already on its device in bf16 (full weights are dropped layer by layer
        as they are sharded; load on CPU / meta and move layer-wise for models that do not fit one GPU)."""
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        self.layers = list(model.get_model().layers)
        self.n_layers = len(self.layers)
        named0 = dict(self.layers[0].named_parameters())
        self.shapes = [tuple(named0[n].shape) for n in self.LAYER_PARAMS]
        extra = set(named0) - set(self.LAYER_PARAMS)
        if extra:
            raise ValueError(f"Zero3Inference: decoder layer has parameters outside the known layout: {sorted(extra)}")
        self.offsets, total = [], 0
        for shp in self.shapes:
            self.offsets.append(total)
            n = 1
            for d in shp:
                n *= d
            total += _round8(n)                       # 16-byte aligned sub-tensors (TMA / uint4 loads)
        self.shard = _round8((total + self.world - 1) // self.world)
        self.padded = self.shard * self.world
        dev = named0[self.LAYER_PARAMS[0]].device
        dt = named0[self.LAYER_PARAMS[0]].dtype
        self.shards = []
        lo = self.rank * self.shard
        for layer in self.layers:
            named = dict(layer.named_parameters())
            flat = torch.zeros(self.padded, dtype=dt, device=dev)
            for name, shp, off in zip(self.LAYER_PARAMS, self.shapes, self.offsets):
                p = named[name]
                if tuple(p.shape) != shp:
                    raise ValueError("Zero3Inference: decoder layers must be shape-homogeneous")
                flat[off:off + p.numel()].copy_(p.data.reshape(-1))
                p.data = torch.empty(0, dtype=dt, device=dev)       # drop the full copy
                p.requires_grad_(False)
            self.shards.append(flat[lo:lo + self.shard].clone())
            del flat
        self.bufs = [torch.empty(self.padded, dtype=dt, device=dev) for _ in range(2)]
        self._slot_of = {}            # layer index -> (staging slot, async handle | None) of an in-flight / landed gather
        self._launched = 0
        self.gathers = 0              # statistics: number of layer gathers issued
        model.get_model()._zero3 = self
        self.model = model

    # ---- gather pipeline ---------------------------------------------------------------------------------------------
    def _gather(self, l: int):
        slot = self._launched % 2
        self._launched += 1
        self.gathers += 1
        buf = self.bufs[slot]
        if self.world > 1:
            # issued on NCCL's stream after everything already enqueued on the compute stream (i.e. after the previous
            # user of this staging slot), so it overlaps the layer that is about to run
            h = dist.all_gather_into_tensor(buf, self.shards[l], group=self.pg, async_op=True)
        else:
            buf[:self.shard].copy_(self.shards[l])
            h = None
        self._slot_of[l] = (slot, h)

    def before_layer(self, i: int):
        """Called by the decoder loop right before layer i runs: make its weights resident, prefetch the next layer."""
        if i not in self._slot_of:
            self._gather(i)                                        # cold start (first forward)
        slot, h = self._slot_of.pop(i)
        if h is not None:
            h.wait()                                               # compute stream waits for the gather
        buf = self.bufs[slot]
        named = dict(self.layers[i].named_parameters())
        for name, shp, off in zip(self.LAYER_PARAMS, self.shapes, self.offsets):
            n = 1
            for d in shp:
                n *= d
            named[name].data = buf[off:off + n].view(shp)
        nxt = (i + 1) % self.n_layers                              # wraps: keeps the pipe full across decode steps
        if nxt not in self._slot_of and self.n_layers > 1:
            self._gather(nxt)

    def all_done(self, done: torch.Tensor) -> bool:
        """Ranks run the layer collectives in lock-step, so generation stops only when EVERY rank is finished."""
        flag = done.all().to(torch.int32).view(1)
        if self.world > 1:
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.pg)
        return bool(flag.item())

    def bytes_per_gpu(self):
        es = self.shards[0].element_size()
        return dict(shards=self.n_layers * self.shard * es, staging=2 * self.padded * es)
