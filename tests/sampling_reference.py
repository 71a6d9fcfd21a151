"""A numpy restatement of the sampling rule of `ops.sample_tokens` (csrc/sample.cu; cambrian_b200/generation.py states it),
written from the rule and not from the kernel: Philox4x32-10, the keep set, and the Gumbel-max race in fp64.  Also a CPU
stand-in of `ops.sample_tokens` for host-logic tests on machines without a GPU.

The reference differs from the kernel only in rounding: expf and logf are fp64 here, so a draw whose top two race keys
are within a relative 1e-4, or whose top-p boundary mass lies within 1e-5 of top_p, may legitimately go the other way.
`race` reports both conditions so a test can set such draws aside and count them."""
from __future__ import annotations

import numpy as np
import torch

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF
MASS_SCALE = 2.0 ** 40


def philox4x32_10(ctr, key):
    """Philox4x32-10 over arrays: ctr uint64 [..., 4] and key [..., 2] holding 32-bit words -> uint64 [..., 4]."""
    c = [np.asarray(ctr[..., j], dtype=np.uint64) for j in range(4)]
    k0 = np.asarray(key[..., 0], dtype=np.uint64)
    k1 = np.asarray(key[..., 1], dtype=np.uint64)
    m = np.uint64(MASK32)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(W0)) & m
            k1 = (k1 + np.uint64(W1)) & m
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m]
    return np.stack(c, -1)


def uniforms(V: int, seed: int, step: int) -> np.ndarray:
    """u_i for i < V: word i & 3 of Philox at key = seed, counter = (i >> 2, step lo, step hi, 0), as
    ((w >> 9) + 0.5) * 2^-23 (fp64, equal to the kernel's exact fp32 value)."""
    seed &= (1 << 64) - 1
    step &= (1 << 64) - 1
    ng = (V + 3) // 4
    ctr = np.zeros((ng, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(ng, dtype=np.uint64)
    ctr[:, 1] = step & MASK32
    ctr[:, 2] = step >> 32
    key = np.array([seed & MASK32, seed >> 32], dtype=np.uint64)
    w = philox4x32_10(ctr, np.broadcast_to(key, (ng, 2))).reshape(-1)[:V]
    return ((w >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def scores(logits_row, T: float) -> np.ndarray:
    """fp32 scores: the row itself at T == 1, else the IEEE fp32 quotient."""
    x = np.asarray(logits_row, dtype=np.float32)
    return x if np.float32(T) == np.float32(1.0) else x / np.float32(T)


def keep_set(s: np.ndarray, k: int, p: float, with_margin: bool = False):
    """The kept mask of fp32 scores s under top_k k and top_p p.  With with_margin, also the distance to p of the
    boundary masses G / Z at the cut, of the lowest kept and the highest dropped distinct score (inf when top-p is off)."""
    V = s.shape[0]
    keep = np.ones(V, dtype=bool)
    if 0 < k < V:
        kth = np.sort(s)[::-1][k - 1]
        keep &= s >= kth
    margin = np.inf
    p32 = float(np.float32(p))
    if p32 < 1.0:
        sk = s[keep].astype(np.float64)
        mass = np.rint(np.exp(sk - sk.max()) * MASS_SCALE)
        z = mass.sum()
        vals, inv = np.unique(sk, return_inverse=True)          # ascending distinct scores
        per = np.bincount(inv, weights=mass, minlength=len(vals))
        greater = np.concatenate([np.cumsum(per[::-1])[::-1][1:], [0.0]])   # mass strictly above each distinct value
        ok = greater < p32 * z
        keep_idx = np.nonzero(keep)[0]
        keep[keep_idx[~ok[inv]]] = False
        # the cut: the lowest kept and the highest dropped distinct score
        lo = np.argmax(ok)
        cut = greater[lo:lo + 1] if lo == 0 else greater[lo - 1:lo + 1]
        margin = float(np.min(np.abs(cut / z - p32)))
    return (keep, margin) if with_margin else keep


def race(logits_row, T: float, k: int, p: float, seed: int, step: int):
    """(token, relative gap of the top two race keys, top-p boundary margin) of one row in fp64."""
    s = scores(logits_row, T)
    keep, margin = keep_set(s, k, p, with_margin=True)
    u = uniforms(s.shape[0], seed, step)
    key = np.where(keep, s.astype(np.float64) - np.log(-np.log(u)), -np.inf)
    order = np.argsort(-key, kind="stable")
    tok = int(order[0])
    gap = np.inf
    if keep.sum() > 1:
        a, b = key[order[0]], key[order[1]]
        gap = float((a - b) / max(1.0, abs(a)))
    return tok, gap, margin


def sample_tokens(logits, temperature, top_k, top_p, seed, step, out=None, workspace=None):
    """CPU stand-in of ops.sample_tokens: the fp64 race per row."""
    rows = logits.shape[0]
    lg = logits.detach().float().cpu().numpy()
    t, k, p = temperature.cpu().tolist(), top_k.cpu().tolist(), top_p.cpu().tolist()
    sd, st = seed.cpu().tolist(), step.cpu().tolist()
    toks = torch.tensor([race(lg[b], t[b], k[b], p[b], sd[b], st[b])[0] for b in range(rows)], dtype=torch.int64)
    if out is None:
        return toks.to(logits.device)
    out.copy_(toks)
    return out


def install(monkeypatch):
    if torch.cuda.is_available():
        raise RuntimeError("the sampling stand-in is for GPU-less machines only: on a GPU the kernel runs")
    from cambrian_b200 import ops
    monkeypatch.setattr(ops, "sample_tokens", sample_tokens)
