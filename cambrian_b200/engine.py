"""Data-parallel training engine for the Cambrian hot path (SURVEY.md §8a A13, §8e).

One process per GPU.  All trainable parameters live in ONE flat bf16 buffer (the compute copy) with matching flat
buffers for bf16 gradients, fp32 master weights and fp32 Adam moments:

  * weight-gradient GEMMs accumulate straight into `param.main_grad` (a view of the flat gradient buffer), so
    autograd never materialises or sums parameter gradients;
  * gradient reduction = one NCCL collective per contiguous BUCKET of the flat gradient buffer, launched asynchronously the
    moment the bucket's last gradient contribution has been enqueued, so NVLink traffic overlaps the remaining backward
    GEMMs.  `zero_stage=0` (DDP, BASELINE config 3) all-reduces the bucket; `zero_stage=2` (BASELINE config 4,
    scripts/zero2.json:16-22) reduce-scatters it — every rank owns the 1/world piece of EVERY bucket, keeps fp32 master /
    Adam state for its pieces only (12 of the 16 bytes per parameter), and all-gathers the updated bf16 pieces in place.
    Frozen towers are never reduced;
  * the optimizer is a fused AdamW kernel over contiguous SEGMENTS of equal hyper-parameters (the reference's parameter
    groups, cambrian_trainer.py:242-381: `mm_projector_lr` / `mm_vision_sampler_lr` group learning rates, no weight decay
    for norm and bias parameters) on a side stream.  `background_optimizer=True` launches it as ONE small block per SM so it
    co-resides with GEMM CTAs; the default is the full-occupancy launch placed where it overlaps the frozen towers of the
    next step, because a slow HBM-bound update that shares HBM with the GEMMs for its whole duration costs them more than
    it saves (measured on an earlier GPU generation; not re-measured on H100);
  * gradient clipping (`max_grad_norm`, HF Trainer's default 1.0 is active in every reference script): per-bucket sums of
    squares are taken as the buckets arrive, the clip coefficient stays on the device (no host sync) and is applied inside
    AdamW.  Because no update may start before the global norm is known, with clipping the updates run after backward, in
    the order the NEXT forward consumes the parameters, and each consumer waits only for its own bucket's event
    (`autograd._await`): the optimizer hides under the frozen towers and the first decoder layers of the next step.
    Without clipping each bucket is updated as soon as it is reduced, under the rest of backward;
  * `offload_optimizer=True` (DeepSpeed's `offload_optimizer`, scripts/zero3_offload.json) keeps the fp32 master and
    moments in registered host memory: the device holds 4 B per trainable parameter instead of 16, and the update kernel
    (`ops.adamw_host`) streams the state over PCIe, same arithmetic on the GPU, same schedule and streams as above.

Gradient contributions are counted per parameter: the counts are structural (one per weight-gradient GEMM site, lm_head
notifies once per step however many row chunks it processes), learned on the first step and verified equal across ranks
before any overlapped launch is allowed — ranks must issue identical collectives in identical order.

The reference does its gradient reduction inside torch_xla FSDP (`xm.all_reduce` helper at cambrian_trainer.py:181-190)
and steps HF Trainer's AdamW (cambrian_trainer.py:242-381).
"""
from __future__ import annotations

import functools
import weakref

import torch
import torch.distributed as dist

from . import ops


def _round_up(n: int, m: int) -> int:
    return (n + m - 1) // m * m


class _EventHandle:
    """`Work.wait()` look-alike for our own collective kernel: makes the CURRENT stream wait for the recorded event."""

    def __init__(self, ev):
        self.ev = ev

    def wait(self):
        torch.cuda.current_stream().wait_event(self.ev)


def cosine_schedule_with_warmup(num_warmup_steps: int, num_training_steps: int, num_cycles: float = 0.5):
    """`lr_lambda` equal to transformers.get_cosine_schedule_with_warmup (the reference scripts train with
    `--lr_scheduler_type cosine --warmup_ratio 0.03`, scripts/cambrian/finetune_cambrian_8b.sh): step -> multiplier."""
    import math

    def f(step: int) -> float:
        if step < num_warmup_steps:
            return float(step) / float(max(1, num_warmup_steps))
        progress = float(step - num_warmup_steps) / float(max(1, num_training_steps - num_warmup_steps))
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * float(num_cycles) * 2.0 * progress)))
    return f


class TrainEngine:
    def __init__(self, model: torch.nn.Module, lr: float = 4e-5, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, bucket_mb: float = 256.0, process_group=None, overlap: bool = True,
                 zero_stage: int = 0, max_grad_norm: float | None = None, mm_projector_lr: float | None = None,
                 mm_vision_sampler_lr: float | None = None, lr_lambda=None, loss_scale: float = 1.0,
                 background_optimizer: bool = False, collective: str = "nccl", offload_optimizer: bool = False):
        if zero_stage not in (0, 2):
            raise ValueError("zero_stage must be 0 or 2")
        if hasattr(model, "check_trainable"):   # a model that trains only in some configurations refuses the others
            model.check_trainable()
        from .quant import quantized_format
        fmt = quantized_format(model)
        if fmt is not None:
            raise ValueError(f"TrainEngine: the model has {fmt} decoder weights, which are inference-only "
                             "(QLoRA training is not supported)")
        if mm_projector_lr is not None and mm_vision_sampler_lr is not None:
            raise AssertionError("mm_projector_lr and mm_vision_sampler_lr are mutually exclusive")  # cambrian_trainer.py:259
        self.model = model
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.max_grad_norm = max_grad_norm if max_grad_norm and max_grad_norm > 0 else None
        self.lr_lambda = lr_lambda            # step (0-based, as torch LambdaLR) -> multiplier of every group's lr
        self.loss_scale = float(loss_scale)   # e.g. 1 / gradient_accumulation_steps; folded into the fused loss gradient
        self.background = background_optimizer
        if collective not in ("nccl", "multimem", "p2p"):
            raise ValueError("collective must be 'nccl', 'multimem' (in-switch NVLS all-reduce kernel) or 'p2p'")
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        self.overlap = overlap
        self.zero_stage = zero_stage
        self.step_count = 0
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        if not named:
            raise ValueError("TrainEngine: model has no trainable parameters")
        dev = named[0][1].device
        self.params = [p for _, p in named]
        self.names = [n for n, _ in named]
        for p in self.params:
            if p.dtype != torch.bfloat16:
                raise ValueError("TrainEngine expects bf16 parameters (fp32 masters are kept by the engine)")
        # ---- parameter groups (cambrian_trainer.py:242-381)
        norm_params = set()
        for m in model.modules():
            if isinstance(m, torch.nn.LayerNorm) or type(m).__name__.endswith("RMSNorm"):
                norm_params.update(id(p) for p in m.parameters(recurse=False))
        self.hparams = []     # per parameter: (group lr, weight decay)
        for n, p in named:
            glr = lr
            if mm_projector_lr is not None and "mm_projector" in n:
                glr = mm_projector_lr
            elif mm_vision_sampler_lr is not None and ("vision_sampler" in n or "vision_query" in n):
                glr = mm_vision_sampler_lr
            decay = weight_decay if (id(p) not in norm_params and "bias" not in n) else 0.0
            self.hparams.append((glr, decay))
        # ---- flat layout + buckets: contiguous parameter ranges of ~bucket_mb; with ZeRO-2 every bucket is padded to a
        #      multiple of 8 * world elements so each rank owns an equal, 16-byte aligned piece of it
        self.collective = collective if (self.world > 1 and zero_stage == 0) else "nccl"
        align = 8 * self.world if (zero_stage == 2 or self.collective != "nccl") else 8
        limit = int(bucket_mb * 1024 * 1024 / 2)
        offs, total = [], 0
        self.buckets = []      # (start_elem, end_elem, [param indices])
        cur, cur_start = [], 0
        for i, p in enumerate(self.params):
            offs.append(total)
            total += _round_up(p.numel(), 8)
            cur.append(i)
            if total - cur_start >= limit:
                total = _round_up(total - cur_start, align) + cur_start
                self.buckets.append((cur_start, total, cur))
                cur, cur_start = [], total
        if cur:
            total = _round_up(total - cur_start, align) + cur_start
            self.buckets.append((cur_start, total, cur))
        self.offsets = offs
        self.total = total
        self.flat_p = torch.zeros(total, dtype=torch.bfloat16, device=dev)
        self._symm = self._comm_stream = None
        if self.collective != "nccl":
            # gradients live in a symmetric allocation every rank maps (and the switch multicasts into): comm.py
            from .comm import SymmetricAllReduce
            import os
            self._symm = SymmetricAllReduce(total, dev, process_group, ctas=int(os.environ.get("CB_AR_CTAS", "0")),
                                            use_multicast=self.collective == "multimem")
            self.flat_g = self._symm.buf
            self._comm_stream = torch.cuda.Stream(device=dev)
        else:
            self.flat_g = torch.zeros(total, dtype=torch.bfloat16, device=dev)
        self._bucket_of = {}
        for b, (_, _, idx) in enumerate(self.buckets):
            for i in idx:
                self._bucket_of[i] = b
        for i, (p, o) in enumerate(zip(self.params, offs)):
            n = p.numel()
            self.flat_p[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.flat_p[o:o + n].view(p.shape)          # re-point: compute copy now lives in the flat buffer
            p.main_grad = self.flat_g[o:o + n].view(p.shape)
            p._cb_fresh = set()
            p._cb_notify = functools.partial(self._on_write, i)
            p._cb_engine = self
            p._cb_bucket = self._bucket_of[i]
            p.grad = None
        # ---- optimizer state: whole buffer (DDP) or this rank's piece of every bucket (ZeRO-2); on the device, or in
        #      registered host memory with offload_optimizer
        self.offload = bool(offload_optimizer)
        self._closed = False
        self._host_finalizer = None
        self.piece_base = None
        if zero_stage == 2:
            self.piece_base, n_state = [], 0
            for (s, e, _) in self.buckets:
                self.piece_base.append(n_state)
                n_state += (e - s) // self.world
            self.shard = n_state
            if not self.offload:
                self.master = torch.empty(n_state, dtype=torch.float32, device=dev)
                for b, (s, e, _) in enumerate(self.buckets):
                    lo, hi = self._piece(b)
                    self.master[self.piece_base[b]:self.piece_base[b] + hi - lo].copy_(self.flat_p[lo:hi])
            self.shard_g = torch.zeros(n_state, dtype=torch.bfloat16, device=dev)
        else:
            self.shard = 0
            n_state = total
            if not self.offload:
                self.master = self.flat_p.float()
        if self.offload:
            self._init_host_state(n_state)
        else:
            self.exp_avg = torch.zeros(n_state, dtype=torch.float32, device=dev)
            self.exp_avg_sq = torch.zeros(n_state, dtype=torch.float32, device=dev)
        self._static_segments = [self._segments(b, ()) for b in range(len(self.buckets))]
        # ---- clipping state (device side; no host sync)
        self._sumsq = torch.zeros(1, dtype=torch.float32, device=dev)   # reset by the clip kernel itself (stream-ordered)
        self._coef = torch.ones(2, dtype=torch.float32, device=dev)     # [gradient scale incl. 1/world, grad norm]
        self._sumsq_ws = None
        self._sumsq_done = [False] * len(self.buckets)
        # ---- contribution accounting for the backward / collective overlap
        self._expected = None                      # writes per parameter per step, learned on the first step
        self._overlap_ok = False                   # set once the counts were verified equal on every rank
        self._writes = [0] * len(self.params)
        self._remaining = None                     # per bucket: parameters not yet final
        self._launched = [False] * len(self.buckets)
        self._reduced_on_opt = [False] * len(self.buckets)   # opt stream already ordered after bucket's collective
        self._updated = [False] * len(self.buckets)
        self._handles = {}
        self._opt_stream = None
        self._ready = {}                           # bucket -> CUDA event: updated (and all-gathered) parameters visible
        self._use_order = []                       # buckets in the order the forward first touches them (learned, step 1)
        self._use_seen = set()
        self._no_grad = ()
        self._towers_trainable = any("vision_tower" in n for n in self.names)
        # opt-in (bench / training loops): do not make the main stream wait for the optimizer stream at the end of step();
        # every consumer waits for its own bucket instead (autograd._await) — anyone reading parameters by other means
        # right after step() must call wait_for_params()
        self.defer_param_sync = False
        if hasattr(model, "prepare_inputs_labels_for_multimodal"):
            model._cb_param_sync = self.wait_for_params     # kept for API compatibility: a full wait
            model._cb_loss_scale = self.loss_scale

    def _init_host_state(self, n_state):
        """fp32 master and moments as CPU tensors, registered with CUDA when the model is on the GPU (offload_optimizer).
        The master is filled one bucket (ZeRO-2: one piece) at a time through a device scratch of that size: a full-size
        fp32 copy on the device is exactly what offloading exists to avoid."""
        self.master = torch.empty(n_state, dtype=torch.float32)
        self.exp_avg = torch.zeros(n_state, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(n_state, dtype=torch.float32)
        if self.flat_p.is_cuda:
            registered = []
            try:
                for t in (self.master, self.exp_avg, self.exp_avg_sq):
                    registered.append(ops.host_register(t))
            except Exception:
                _release_host_state(self.flat_p.device, registered)
                raise
            # unregisters before the tensors can be freed: on close() or when the engine is collected
            self._host_finalizer = weakref.finalize(self, _release_host_state, self.flat_p.device, registered)
        pieces = [self._piece(b) if self.zero_stage == 2 else self.buckets[b][:2] for b in range(len(self.buckets))]
        scratch = torch.empty(max(hi - lo for lo, hi in pieces), dtype=torch.float32, device=self.flat_p.device)
        for b, (lo, hi) in enumerate(pieces):
            at = self.piece_base[b] if self.zero_stage == 2 else lo
            sc = scratch[:hi - lo]
            sc.copy_(self.flat_p[lo:hi])
            self.master[at:at + hi - lo].copy_(sc)

    # ---- layout helpers --------------------------------------------------------------------------------------------
    def _piece(self, b):
        s, e, _ = self.buckets[b]
        n = (e - s) // self.world
        return s + self.rank * n, s + (self.rank + 1) * n

    def _segments(self, b, skip):
        """Maximal runs [lo, hi) of bucket b with equal (lr, weight decay), leaving out parameters in `skip` (no gradient
        this step: torch.optim skips them entirely)."""
        s, e, idx = self.buckets[b]
        segs = []
        for i in idx:
            if i in skip:
                continue
            lo = self.offsets[i]
            hi = lo + _round_up(self.params[i].numel(), 8)
            hp = self.hparams[i]
            if segs and segs[-1][1] == lo and segs[-1][2] == hp:
                segs[-1] = (segs[-1][0], hi, hp)
            else:
                segs.append((lo, hi, hp))
        return segs

    # ---- per-step protocol ---------------------------------------------------------------------------------------
    def zero_grad(self):
        for p in self.params:
            p._cb_fresh.clear()
            p.grad = None
        self._writes = [0] * len(self.params)
        self._launched = [False] * len(self.buckets)
        self._reduced_on_opt = [False] * len(self.buckets)
        self._updated = [False] * len(self.buckets)
        self._handles = {}
        self._no_grad = ()
        self._sumsq_done = [False] * len(self.buckets)
        if self._expected is not None:
            self._remaining = [sum(1 for i in idx if self._expected[i] > 0) for (_, _, idx) in self.buckets]

    def _opt(self):
        if self._opt_stream is None and self.flat_p.is_cuda:
            self._opt_stream = torch.cuda.Stream(device=self.flat_p.device)
        return self._opt_stream

    def _launch_bucket(self, b):
        """Issue bucket b's gradient collective (asynchronously; NCCL orders it after the work already enqueued on the
        current stream)."""
        s, e, _ = self.buckets[b]
        self._launched[b] = True
        if self.world == 1:
            return
        if self._symm is not None:
            cs = self._comm_stream
            cs.wait_stream(torch.cuda.current_stream())        # after the bucket's last gradient write
            with torch.cuda.stream(cs):
                self._symm.all_reduce_(s, e)
                ev = torch.cuda.Event()
                ev.record(cs)
            self._handles[b] = _EventHandle(ev)
            return
        if self.zero_stage == 2:
            lo, hi = self._piece(b)
            out = self.shard_g[self.piece_base[b]:self.piece_base[b] + hi - lo]
            if dist.get_backend(self.pg) == "nccl":
                self._handles[b] = dist.reduce_scatter_tensor(out, self.flat_g[s:e], op=dist.ReduceOp.SUM, group=self.pg,
                                                              async_op=True)
            else:   # gloo (CPU tests) has no reduce_scatter_tensor: all-reduce the bucket, keep the local piece
                dist.all_reduce(self.flat_g[s:e], op=dist.ReduceOp.SUM, group=self.pg)
                out.copy_(self.flat_g[lo:hi])
        else:
            self._handles[b] = dist.all_reduce(self.flat_g[s:e], op=dist.ReduceOp.SUM, group=self.pg, async_op=True)

    def _grads_of(self, b):
        """(reduced gradient tensor of this rank's part of bucket b, flat offset of its first element)."""
        s, e, _ = self.buckets[b]
        if self.zero_stage == 2:
            lo, hi = self._piece(b)
            if self.world == 1:
                return self.flat_g[lo:hi], lo
            return self.shard_g[self.piece_base[b]:self.piece_base[b] + hi - lo], lo
        return self.flat_g[s:e], s

    def _after_reduce(self, b, side: bool):
        """Order the consumer stream after bucket b's collective (side stream) or after its gradients (world 1)."""
        st = self._opt() if side else None
        if st is not None:
            if b in self._handles:
                with torch.cuda.stream(st):
                    self._handles.pop(b).wait()
            elif not self._reduced_on_opt[b]:
                st.wait_stream(torch.cuda.current_stream())
            self._reduced_on_opt[b] = True
        elif b in self._handles:
            self._handles.pop(b).wait()
        return st

    def _accumulate_sumsq(self, b, side: bool):
        self._sumsq_done[b] = True
        g, _ = self._grads_of(b)
        st = self._after_reduce(b, side)
        if self._sumsq_ws is None:
            self._sumsq_ws = torch.empty(4096, dtype=torch.float32, device=g.device)
        if st is not None:
            with torch.cuda.stream(st):
                ops.sumsq_accumulate(g, self._sumsq, self._sumsq_ws, background=self.background)
        else:
            ops.sumsq_accumulate(g, self._sumsq, self._sumsq_ws, background=self.background)

    def _update_bucket(self, b, side: bool):
        """Fused AdamW over bucket b's segments (this rank's piece under ZeRO-2), then the in-place all-gather of the updated
        bf16 piece (ZeRO-2), then the bucket's `ready` event."""
        self._updated[b] = True
        s, e, _ = self.buckets[b]
        st = self._after_reduce(b, side)
        g, g0 = self._grads_of(b)
        lo_p, hi_p = (self._piece(b) if self.zero_stage == 2 else (s, e))
        state0 = self.piece_base[b] - lo_p if self.zero_stage == 2 else 0     # flat offset -> optimizer-state offset
        segs = self._static_segments[b] if not self._no_grad else self._segments(b, self._no_grad)
        mult = self.lr_lambda(self.step_count) if self.lr_lambda is not None else 1.0
        coef = self._coef if self.max_grad_norm is not None else None

        def run():
            for (lo, hi, (glr, wd)) in segs:
                lo, hi = max(lo, lo_p), min(hi, hi_p)
                if hi <= lo:
                    continue
                self._adamw(self.master[state0 + lo:state0 + hi], self.exp_avg[state0 + lo:state0 + hi],
                            self.exp_avg_sq[state0 + lo:state0 + hi], g[lo - g0:hi - g0], self.flat_p[lo:hi],
                            glr * mult, wd, self.step_count + 1, coef)
            if self.zero_stage == 2 and self.world > 1:
                # in-place all-gather: this rank's piece already sits at its slot of the bucket (NCCL's in-place layout)
                src = self.flat_p[lo_p:hi_p]
                if dist.get_backend(self.pg) != "nccl":
                    src = src.clone()
                h = dist.all_gather_into_tensor(self.flat_p[s:e], src, group=self.pg, async_op=True)
                if h is not None:
                    h.wait()
            if st is not None:
                ev = torch.cuda.Event()
                ev.record(st)
                self._ready[b] = ev

        with ops.nvtx(f"optimizer.bucket{b}"):
            if st is not None:
                with torch.cuda.stream(st):
                    run()
            else:
                run()

    def _adamw(self, master, m, v, g, p16, lr, wd, step, coef):
        if self.offload:
            ops.adamw_host(master, m, v, g, p16, lr, self.betas[0], self.betas[1], self.eps, wd, step,
                           grad_scale=1.0 / self.world, clip_coef=coef)
            return
        ops.adamw(master, m, v, g, p16, lr, self.betas[0], self.betas[1], self.eps, wd, step,
                  grad_scale=1.0 / self.world, clip_coef=coef, background=self.background)

    def _on_write(self, i):
        """Called (host side, in stream order) right after a gradient contribution of parameter i was enqueued."""
        self._writes[i] += 1
        if self._expected is None or not self._overlap_ok:
            return
        if self._writes[i] > self._expected[i]:
            b = self._bucket_of[i]
            if self._launched[b]:
                raise RuntimeError(
                    f"TrainEngine: parameter {self.names[i]} received gradient contribution #{self._writes[i]} after its "
                    f"bucket had been reduced (learned count {self._expected[i]}): the graph changed between steps — call "
                    "engine.relearn() before the step that changes it")
            return
        if self._writes[i] == self._expected[i]:
            b = self._bucket_of[i]
            self._remaining[b] -= 1
            if self._remaining[b] == 0 and not self._launched[b]:
                # a bucket whose parameters also receive plain-autograd gradients is only final at step()
                if all(self._expected[j] > 0 for j in self.buckets[b][2]):
                    self._launch_bucket(b)
                    if self.max_grad_norm is not None:
                        self._accumulate_sumsq(b, side=True)
                    else:
                        self._update_bucket(b, side=True)

    def relearn(self):
        """Forget the learned contribution counts (the next step runs without overlap and re-learns them)."""
        self._expected = None
        self._overlap_ok = False

    def _finalize_unwritten(self):
        """Fold in gradients that reached a parameter through plain autograd (a parameter used by an ordinary torch
        view/op, e.g. the `vision_query[g:g+1]` slice); parameters that received no gradient at all this step are left out
        of the update (as torch.optim does) and their gradient slot is zeroed so the norm / collective see zeros."""
        skip = []
        for i, p in enumerate(self.params):
            if self._launched[self._bucket_of[i]]:
                continue
            if p.grad is not None:
                if p._cb_fresh:
                    p.main_grad.add_(p.grad.to(p.main_grad.dtype))
                else:
                    p.main_grad.copy_(p.grad)
                    p._cb_fresh.add("all")
                p.grad = None
            if not p._cb_fresh:
                p.main_grad.zero_()
                skip.append(i)
        self._no_grad = frozenset(skip)

    def reduce_gradients(self):
        """Launch the collective of every bucket that was not launched during backward (in a fixed order, identical on
        every rank) and, for DDP without an optimizer attached to the call, wait for all of them."""
        for b in reversed(range(len(self.buckets))):
            if not self._launched[b]:
                self._launch_bucket(b)
        if self.world > 1 and self.zero_stage == 0:
            for b in list(self._handles):
                if not self._updated[b] and not self._reduced_on_opt[b]:
                    self._handles.pop(b).wait()

    def _learn_counts(self):
        self._expected = list(self._writes)
        ok = True
        if self.world > 1:
            dev = self.flat_p.device
            t = torch.tensor(self._expected, dtype=torch.int64, device=dev)
            lo, hi = t.clone(), t.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=self.pg)
            dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=self.pg)
            ok = bool(torch.equal(lo, hi))     # one host sync, once
        self._overlap_ok = self.overlap and ok
        if self.overlap and not ok:
            import warnings
            warnings.warn("TrainEngine: gradient-contribution counts differ between ranks; collectives stay serial")

    def step(self):
        if self._closed:
            raise RuntimeError("TrainEngine: step() after close(): the host-resident optimizer state was released")
        first = self._expected is None
        self._finalize_unwritten()
        if first:
            self._learn_counts()
        elif self._overlap_ok and self.world > 1 and self._writes != self._expected:
            # another rank may have launched (or not launched) this parameter's bucket during backward: the ranks' NCCL
            # call sequences can no longer be assumed identical — fail loudly instead of hanging or mixing buckets
            i = next(j for j, (w, x) in enumerate(zip(self._writes, self._expected)) if w != x)
            raise RuntimeError(f"TrainEngine: {self.names[i]} received {self._writes[i]} gradient contributions this step, "
                               f"{self._expected[i]} were learned on step 1; call engine.relearn() before a step whose "
                               "graph differs (it then runs without overlap)")
        side = self.flat_p.is_cuda
        order = list(reversed(range(len(self.buckets))))
        for b in order:                                   # collectives not launched during backward: fixed order
            if not self._launched[b]:
                self._launch_bucket(b)
        if self.max_grad_norm is not None:
            for b in order:
                if not self._sumsq_done[b]:
                    self._accumulate_sumsq(b, side)
            self._clip_coefficient(side)
            upd = [b for b in (self._use_order or range(len(self.buckets)))]
            upd += [b for b in range(len(self.buckets)) if b not in set(upd)]
        else:
            upd = order
        for b in upd:
            if not self._updated[b]:
                self._update_bucket(b, side)
        self.step_count += 1
        if self._opt_stream is not None:
            if self.defer_param_sync and not self._towers_trainable:
                pass        # consumers wait per bucket (autograd._await); wait_for_params() is the full barrier
            else:
                self.wait_for_params()

    def _clip_coefficient(self, side):
        st = self._opt() if side else None
        if self.world > 1 and self.zero_stage == 2:
            # every rank holds the squares of its pieces only
            if st is not None:
                torch.cuda.current_stream().wait_stream(st)
            dist.all_reduce(self._sumsq, op=dist.ReduceOp.SUM, group=self.pg)
            if st is not None:
                st.wait_stream(torch.cuda.current_stream())
        if st is not None:
            with torch.cuda.stream(st):
                ops.clip_coef(self._sumsq, self.max_grad_norm, 1.0 / self.world, self._coef)
        else:
            ops.clip_coef(self._sumsq, self.max_grad_norm, 1.0 / self.world, self._coef)

    def grad_norm(self) -> float:
        """Global L2 norm of the rank-averaged gradient of the last clipped step (host sync; logging only)."""
        return float(self._coef[1].item())

    # ---- parameter readiness ---------------------------------------------------------------------------------------
    def await_bucket(self, b):
        """Make the current stream wait for bucket b's pending update (no-op when none is pending)."""
        if b not in self._use_seen:
            self._use_seen.add(b)
            self._use_order.append(b)
        ev = self._ready.pop(b, None)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def wait_for_params(self):
        """Make the current stream wait for every optimizer update still running on the side stream."""
        if self._opt_stream is not None and self._ready:
            torch.cuda.current_stream().wait_stream(self._opt_stream)
            self._ready.clear()

    # ---- convenience ---------------------------------------------------------------------------------------------
    def train_step(self, **batch):
        self.zero_grad()
        out = self.model(**batch)
        out.loss.backward()
        self.step()
        return out.loss

    def state_bytes(self):
        """Device bytes of training state: bf16 weights and gradients, plus the fp32 master and moments unless offloaded."""
        opt = (self.shard if self.zero_stage == 2 else self.total) * 12
        return self.total * 4 + (0 if self.offload else opt)

    def host_state_bytes(self):
        """Host bytes of the offloaded fp32 master and moments (0 without offload_optimizer)."""
        return 3 * 4 * self.master.numel() if self.offload else 0

    def close(self):
        """Unregister the host-resident optimizer state (after the device has finished with it).  Idempotent, and run
        when the engine is garbage-collected; step() raises afterwards.  The host tensors stay readable."""
        self._closed = True
        if self._host_finalizer is not None:
            self._host_finalizer()


def _release_host_state(device, tensors):
    torch.cuda.synchronize(device)          # no update may still be reading or writing them
    for t in tensors:
        ops.host_unregister(t)
