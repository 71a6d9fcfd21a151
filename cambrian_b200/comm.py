"""Symmetric-memory gradient buffer + in-switch all-reduce (csrc/collective.cu) for the data-parallel engine.

torch.distributed._symmetric_memory is used as PLUMBING only: it allocates the flat bf16 gradient buffer with a fabric /
IPC-shareable handle, exchanges the handles between the ranks of one node and maps (a) every peer's buffer and (b) the NVLS
multicast view of all of them into this process.  The reduction itself is our kernel (`cb_allreduce_symm_bf16`:
`multimem.ld_reduce` / `multimem.st` — the NVSwitch sums and fans out — or peer loads / stores when the fabric has no
multicast), launched per gradient bucket on a dedicated stream ordered after the bucket's last gradient write."""
from __future__ import annotations

import ctypes

import torch
import torch.distributed as dist

from . import _lib
from ._lib import check

FLAG_WORDS = 160 * 8         # AR_MAX_CTAS x AR_MAX_RANKS (collective.cu)


class SymmetricAllReduce:
    def __init__(self, numel: int, device, group=None, ctas: int = 0, use_multicast: bool = True):
        import torch.distributed._symmetric_memory as symm
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        if self.world > 8:
            raise ValueError("SymmetricAllReduce covers one NVSwitch domain (<= 8 ranks)")
        self.buf = symm.empty(numel, dtype=torch.bfloat16, device=device)
        self.buf.zero_()
        self.flags = symm.empty(FLAG_WORDS, dtype=torch.int32, device=device)
        self.flags.zero_()
        torch.cuda.synchronize(device)
        hb = symm.rendezvous(self.buf, self.group)
        hf = symm.rendezvous(self.flags, self.group)
        self._handles = (hb, hf)                         # keep the mappings alive
        self.buf_ptrs = (ctypes.c_uint64 * self.world)(*[int(p) for p in hb.buffer_ptrs])
        self.flag_ptrs = (ctypes.c_uint64 * self.world)(*[int(p) for p in hf.buffer_ptrs])
        mc = int(getattr(hb, "multicast_ptr", 0) or 0)
        self.multicast = mc if use_multicast else 0
        # 128-thread CTAs that share SMs with the GEMM CTAs: one per SM keeps enough switch round trips in flight at any
        # world size (each GPU moves 1/world of a bucket through its own loads / stores)
        self.ctas = int(ctas) if ctas else _lib.load().cb_sm_count()
        self.epoch = 1
        dist.barrier(group=self.group)                   # every rank's flags are zero before anyone raises one

    def all_reduce_(self, start: int, end: int):
        """In-place sum over ranks of buf[start:end] (elements), on the CURRENT stream; (end - start) * 2 bytes must be a
        multiple of 16 * world.  Every rank must call this with the same ranges in the same order."""
        check(_lib.load().cb_allreduce_symm_bf16(self.multicast, ctypes.addressof(self.buf_ptrs), ctypes.addressof(self.flag_ptrs),
                                                 2 * start, 2 * (end - start), self.rank, self.world, self.epoch, self.ctas,
                                                 torch.cuda.current_stream().cuda_stream), "cb_allreduce_symm_bf16")
        self.epoch += 2
