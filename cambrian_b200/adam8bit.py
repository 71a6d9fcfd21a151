"""8-bit AdamW moments (`TrainEngine(optim="adamw_bnb_8bit")`, HF's `--optim adamw_bnb_8bit`: cambrian_trainer.py:365-380).

The format follows bitsandbytes' block-wise 8-bit optimizer state; this module is the one place on the host that states
it (the kernels in csrc/adam8bit.cu are the other side).  Per trainable parameter that keeps 8-bit moments:

  * blocks of BLOCK = 256 consecutive elements of the parameter (the last block may be partial); per block and moment one
    fp32 scale absmax = max |x| over the block;
  * the first moment m is coded against the signed dynamic map (`quant.dynamic_map()`, bitsandbytes
    `create_dynamic_map(signed=True)`), the second moment v against the unsigned one (`quant.dynamic_map(signed=False)`);
  * code = the map entry nearest x * (1 / absmax): the first entry >= that value or the one before it, whichever is closer
    in fp32, the larger one on a tie (quant.py's rule); an all-zero block stores the code of 0.0;
  * dequantisation: map[code] * absmax (one rounding).

One step, per element: dequantise m and v; update them in fp32; update the fp32 master with the updated, unquantised m and
v with exactly the arithmetic of the fp32-moment kernel (same roundings, the device clip coefficient, `grad_scale`);
write the bf16 copy; then take each block's new absmax of m and of v and requantise both.

Which parameters keep fp32 moments (`fp32_moments`): those with fewer than MIN_8BIT_SIZE = 4096 elements (bitsandbytes'
`min_8bit_size`) and every `nn.Embedding` weight (current HF Trainer registers a 32-bit override for each embedding when
the optimizer is bitsandbytes' 8-bit one).  They go through the fp32-moment kernels unchanged.

Deviations from bitsandbytes:
  * bitsandbytes updates a bf16 parameter in place; the engine keeps its fp32 master, so only the moments change format;
  * the block size of 256 is bitsandbytes' block-wise optimizer's as we understand it; no byte compatibility with its
    optimizer state dicts is claimed (the engine saves no optimizer state).
"""
from __future__ import annotations

import torch

from .quant import dynamic_map

BLOCK = 256
MIN_8BIT_SIZE = 4096

# HF TrainingArguments.optim names -> 8-bit moments or not
OPTIM_8BIT = ("adamw_bnb_8bit", "adamw_8bit")
OPTIM_32BIT = ("adamw_torch",)


def signed_map() -> torch.Tensor:
    """The first moment's 256 sorted code values."""
    return dynamic_map(signed=True)


def unsigned_map() -> torch.Tensor:
    """The second moment's 256 sorted code values."""
    return dynamic_map(signed=False)


def resolve_optim(optim: str) -> bool:
    """True for 8-bit moments, False for fp32 moments; refuses the rest."""
    if optim in OPTIM_8BIT:
        return True
    if optim in OPTIM_32BIT:
        return False
    if optim == "paged_adamw_8bit":
        raise NotImplementedError("optim='paged_adamw_8bit': paged optimizer state is not supported; "
                                  "use optim='adamw_bnb_8bit' with offload_optimizer=True to keep the state in host memory")
    raise ValueError(f"optim={optim!r}: expected one of {OPTIM_32BIT + OPTIM_8BIT}")


def embedding_params(model) -> set:
    """ids of every `nn.Embedding` weight of `model`."""
    return {id(m.weight) for m in model.modules() if isinstance(m, torch.nn.Embedding)}


def fp32_moments(p: torch.Tensor, embeddings: set) -> bool:
    """True when parameter p keeps fp32 moments in 8-bit mode."""
    return p.numel() < MIN_8BIT_SIZE or id(p) in embeddings


def blocks(n: int) -> int:
    """Blocks (scales per moment) of an n-element 8-bit range."""
    return (n + BLOCK - 1) // BLOCK
