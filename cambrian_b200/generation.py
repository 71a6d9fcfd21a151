"""Host-side decoding policy for `CambrianLlamaForCausalLM.generate` — the part of HF `GenerationMixin.generate` the
reference's callers use (cambrian_llama.py:437-483 forwards **kwargs to it; callers: inference.py:77-85,
cambrian/serve/model_worker.py:177-187, eval/eval/*/*_eval.py): greedy / temperature + top-k + top-p sampling, EOS and
user `stopping_criteria`, `streamer`, `max_new_tokens` / `max_length`.

Every keyword is either honoured or rejected with an exception naming it — nothing is silently dropped.

Sampling (`do_sample=True`) on CUDA logits runs one kernel, `ops.sample_tokens` (csrc/sample.cu), for all rows of a step;
`generate()` runs it inside its decode CUDA graph and the server (serving.py) inside each bucket's graph.  The rule:
  * scores s = logits when temperature == 1, else logits / temperature (IEEE division);
  * top-k (0 < top_k < V): keep s_i >= the k-th largest score, ties kept (the set `warp_logits` keeps);
  * top-p (< 1): over the kept scores, keep i iff the softmax mass of the kept scores strictly greater than s_i is below
    top_p.  The mass is exp(s - max) in fp32, rounded to an integer multiple of 2^-40 and summed exactly, so no summation
    order enters.  This is HF's rule (sorted ascending, `cumsum <= 1 - top_p` removed) restated, except that a tie at the
    boundary is kept whole where HF's unstable sort keeps an arbitrary part of it;
  * draw: the exponential race that torch.multinomial uses (Gumbel-max): the kept i with the largest s_i - log(-log u_i),
    the lowest index on a tie, where u_i comes from Philox4x32-10 keyed by the row's 64-bit seed at counter
    (i >> 2, step) and has 23 random bits, strictly inside (0, 1).
  * seeds: one 64-bit seed S per generate() call, drawn from `generator` (or the default generator of the logits' device)
    at the first sampled token; row b uses S + b, and token t of a row (t = 0 for the prefill's token) uses step t.  A
    served request gets the seed row 0 of a solo generate() with the same generator gets.
So a row's token is a function of its logits, its parameters, its seed and its step alone: the same generator gives the
same tokens run after run, whatever rows are sampled beside it.  These are not the tokens torch.multinomial's stream
drew for the same generator before this kernel existed; the distribution is the same warped softmax.

CPU logits keep the torch path: `warp_logits` (HF's warpers) and torch.multinomial with `generator`."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional

import torch

from . import ops

# keywords of HF generate that only make sense with features this path does not implement: rejected when they would
# change the result, accepted when they carry their neutral value
_NEUTRAL = {"num_beams": 1, "num_beam_groups": 1, "num_return_sequences": 1, "repetition_penalty": 1.0, "length_penalty": 1.0,
            "no_repeat_ngram_size": 0, "penalty_alpha": None, "typical_p": 1.0, "epsilon_cutoff": 0.0, "eta_cutoff": 0.0,
            "diversity_penalty": 0.0, "encoder_repetition_penalty": 1.0, "bad_words_ids": None, "force_words_ids": None,
            "constraints": None, "prefix_allowed_tokens_fn": None, "logits_processor": None, "assistant_model": None,
            "output_attentions": False, "output_hidden_states": False, "output_scores": False, "output_logits": False,
            "return_dict_in_generate": False, "synced_gpus": False, "min_p": None, "suppress_tokens": None,
            "begin_suppress_tokens": None, "forced_bos_token_id": None, "forced_eos_token_id": None, "renormalize_logits": False,
            "use_cache": True, "min_length": 0, "min_new_tokens": None, "early_stopping": False, "negative_prompt_ids": None,
            "cache_implementation": None, "guidance_scale": None, "sequence_bias": None, "exponential_decay_length_penalty": None}


@dataclass
class GenerationArgs:
    max_new_tokens: int = 32
    do_sample: bool = False
    temperature: float = 1.0
    top_k: int = 50            # HF GenerationConfig default, applied whenever do_sample=True (as in the reference's callers)
    top_p: float = 1.0
    eos_token_ids: List[int] = field(default_factory=list)
    pad_token_id: int = 0
    stopping_criteria: List[Callable] = field(default_factory=list)
    streamer: Optional[object] = None
    generator: Optional[torch.Generator] = None
    seed: Optional[int] = None  # the sampling seed S, drawn at the first sampled token (draw_seed)
    step: int = 0               # the index of the next sampled token of the eager loop

    @classmethod
    def from_kwargs(cls, model, prompt_len: int, kwargs: dict):
        kw = dict(kwargs)
        gc = kw.pop("generation_config", None) or getattr(model, "generation_config", None)

        def take(name, default):
            if name in kw:
                return kw.pop(name)
            v = getattr(gc, name, None) if gc is not None else None
            return default if v is None else v

        a = cls()
        max_new = kw.pop("max_new_tokens", None)
        max_len = kw.pop("max_length", None)
        if max_new is None and max_len is not None:
            max_new = int(max_len) - prompt_len              # HF: max_length counts the prompt
            if max_new < 1:
                raise ValueError(f"max_length={max_len} leaves no room after a prompt of {prompt_len} positions")
        if max_new is None:
            max_new = getattr(gc, "max_new_tokens", None) or 32
        a.max_new_tokens = int(max_new)
        a.temperature = float(take("temperature", 1.0))
        a.do_sample = bool(take("do_sample", False))
        if a.do_sample and a.temperature in (0, 0.0):
            a.do_sample = False                               # inference.py:81 passes temperature=0 with do_sample=False
        if a.do_sample and a.temperature < 0:
            raise ValueError("`temperature` has to be a strictly positive float")
        a.top_k = int(take("top_k", 50) or 0)
        a.top_p = float(take("top_p", 1.0))
        if not 0.0 < a.top_p <= 1.0:
            raise ValueError(f"`top_p` has to be a float > 0 and <= 1, but is {a.top_p}")
        eos = take("eos_token_id", getattr(model.config, "eos_token_id", None))
        a.eos_token_ids = [int(e) for e in (eos if isinstance(eos, (list, tuple)) else ([] if eos is None else [eos]))]
        pad = take("pad_token_id", getattr(model.config, "pad_token_id", None))
        a.pad_token_id = int(pad) if pad is not None else (a.eos_token_ids[0] if a.eos_token_ids else 0)
        sc = kw.pop("stopping_criteria", None)
        a.stopping_criteria = list(sc) if sc is not None else []
        a.streamer = kw.pop("streamer", None)
        a.generator = kw.pop("generator", None)
        kw.pop("bos_token_id", None)                          # irrelevant here: decoding starts from the prompt embeddings
        for name, neutral in _NEUTRAL.items():
            if name in kw:
                v = kw.pop(name)
                if v != neutral and not (neutral is None and not v) and not (name == "use_cache" and v is None):
                    raise NotImplementedError(f"generate(): `{name}={v!r}` is not supported by the cambrian_b200 decoder "
                                              f"(only its neutral value {neutral!r})")
        if kw:
            raise TypeError(f"generate(): unexpected keyword argument(s) {sorted(kw)} (neither implemented nor ignorable)")
        return a


def warp_logits(logits: torch.Tensor, temperature: float, top_k: int, top_p: float) -> torch.Tensor:
    """HF's sampling warpers in their order (TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper with
    min_tokens_to_keep=1): returns fp32 scores with filtered entries at -inf."""
    scores = logits.float()
    if temperature != 1.0:
        scores = scores / temperature
    V = scores.shape[-1]
    if top_k and 0 < top_k < V:
        kth = torch.topk(scores, top_k, dim=-1).values[..., -1, None]
        scores = scores.masked_fill(scores < kth, float("-inf"))
    if top_p < 1.0:
        sorted_logits, sorted_idx = torch.sort(scores, descending=False, dim=-1)
        cum = sorted_logits.softmax(-1).cumsum(-1)
        remove = cum <= (1.0 - top_p)
        remove[..., -1:] = False                              # min_tokens_to_keep = 1
        scores = scores.masked_fill(remove.scatter(-1, sorted_idx, remove), float("-inf"))
    return scores


def draw_seed(args: GenerationArgs, device) -> int:
    """The call's 64-bit sampling seed S, drawn once from args.generator (or the default generator of `device`)."""
    if args.seed is None:
        g = args.generator
        lo, hi = torch.randint(0, 1 << 32, (2,), generator=g, device=g.device if g is not None else device).tolist()
        args.seed = lo | hi << 32
    return args.seed


def as_int64(v: int) -> int:
    """A uint64 value as the int64 with the same bits (the seed buffers are int64 tensors)."""
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >= 1 << 63 else v


def sampling_params(args: GenerationArgs, rows: int, device):
    """(temperature, top_k, top_p, seed, step) device tensors of ops.sample_tokens for `rows` rows of one call: seed
    S + b for row b, step args.step."""
    S = draw_seed(args, device)
    return (torch.full((rows,), args.temperature, dtype=torch.float32, device=device),
            torch.full((rows,), min(args.top_k, (1 << 31) - 1), dtype=torch.int32, device=device),
            torch.full((rows,), args.top_p, dtype=torch.float32, device=device),
            torch.tensor([as_int64(S + b) for b in range(rows)], dtype=torch.int64, device=device),
            torch.full((rows,), args.step, dtype=torch.int64, device=device))


def next_tokens(logits: torch.Tensor, args: GenerationArgs) -> torch.Tensor:
    if not args.do_sample:
        return logits.argmax(-1)
    if not logits.is_cuda:
        probs = warp_logits(logits, args.temperature, args.top_k, args.top_p).softmax(-1)
        return torch.multinomial(probs, 1, generator=args.generator).squeeze(-1)
    tok = ops.sample_tokens(logits, *sampling_params(args, logits.shape[0], logits.device))
    args.step += 1
    return tok


def should_stop(args: GenerationArgs, generated: torch.Tensor, scores, done: torch.Tensor) -> torch.Tensor:
    """Apply EOS and the user's stopping criteria to the tokens generated so far ([B, t], as HF hands them over when
    generation starts from inputs_embeds).  Criteria may return a bool or a [B] bool tensor (HF >= 4.39)."""
    last = generated[:, -1]
    for e in args.eos_token_ids:
        done = done | (last == e)
    for crit in args.stopping_criteria:
        r = crit(generated, scores)
        if torch.is_tensor(r):
            done = done | r.to(done.device).bool().reshape(-1).expand_as(done)
        elif r:
            done = torch.ones_like(done)
    return done
