"""Torch reference of the paged decode KV cache (cambrian_b200/paged_kv.py states the definition): gather a row's pages,
then a dense softmax in fp64 (FP8 pages dequantised by the kv_fp8.py rule).  CPU stand-ins of the two entry points for
host-logic tests are built from it; they refuse to install in a process that can see a GPU."""
import torch

import kv_fp8_reference as KR


def gather(pages, table_row, L, page_size):
    """Positions [0, L) of one row: [L, ...] from pages [num_pages, page_size, ...] through its block-table row."""
    raw = pages.view(torch.uint8) if pages.dtype == torch.float8_e4m3fn else pages
    idx = torch.arange(max(L, 0))
    out = raw[table_row[idx // page_size].long(), idx % page_size]
    return out.view(pages.dtype) if raw is not pages else out


def decode_attention(q, kp, vp, ksc, vsc, table, lens, len_add=1, scale=None, dtype=torch.float64):
    """q [rows, nh, hd] -> o [rows, nh, hd] in `dtype`: row b attends over its positions below lens[b] + len_add; an
    inactive (lens < 0) or empty row gives zeros.  fp64 is the reference; bf16 mimics eager bf16 (bf16 matmuls, fp32
    softmax rounded to bf16), the yardstick of the parity criterion."""
    rows, nh, hd = q.shape
    ps, nkv = kp.shape[1], kp.shape[2]
    G = nh // nkv
    scale = hd ** -0.5 if scale is None else scale
    out = torch.zeros((rows, nh, hd), dtype=dtype)
    table, lens = table.cpu(), lens.cpu()
    for b in range(rows):
        if int(lens[b]) < 0:
            continue
        L = min(int(lens[b]) + len_add, table.shape[1] * ps)
        if L <= 0:
            continue
        k = gather(kp.cpu(), table[b], L, ps)
        v = gather(vp.cpu(), table[b], L, ps)
        if ksc is not None:
            k = KR.dequantize(k, gather(ksc.cpu(), table[b], L, ps))
            v = KR.dequantize(v, gather(vsc.cpu(), table[b], L, ps))
        k = k.to(dtype).repeat_interleave(G, 1)                                  # [L, nh, hd]
        v = v.to(dtype).repeat_interleave(G, 1)
        s = torch.einsum("hd,thd->ht", q[b].cpu().to(dtype), k) * scale
        p = torch.softmax(s.to(torch.float64 if dtype == torch.float64 else torch.float32), -1).to(dtype)
        out[b] = torch.einsum("ht,thd->hd", p, v)
    return out


# ---- CPU stand-ins of ops.paged_kv_append / ops.attn_decode_paged (host-logic tests on machines without a GPU) ----
def paged_kv_append(k, v, k_pages, v_pages, k_scales, v_scales, block_table, lens=None, offset=0,
                    offset_from_lens=False):
    rows, S = k.shape[:2]
    ps = k_pages.shape[1]
    for b in range(rows):
        if lens is not None and int(lens[b]) < 0:
            continue
        start = int(offset) + (int(lens[b]) if offset_from_lens else 0)
        for s in range(S):
            p = start + s
            page, slot = int(block_table[b, p // ps]), p % ps
            for src, dst, dsc in ((k, k_pages, k_scales), (v, v_pages, v_scales)):
                if dsc is None:
                    dst[page, slot] = src[b, s]
                else:
                    q, sc = KR.quantize_rows(src[b, s].float())
                    dst[page, slot] = q
                    dsc[page, slot] = sc


def attn_decode_paged(q, k_pages, v_pages, k_scales, v_scales, block_table, lens, workspace, *, len_add=1, scale=None):
    o = decode_attention(q[:, 0], k_pages, v_pages, k_scales, v_scales, block_table, lens, len_add, scale)
    return o.to(torch.bfloat16)[:, None]


def attn_decode_paged_workspace(rows, nh, max_pages, page_size, hd, device):
    return torch.empty(1, dtype=torch.float32, device=device)


def install(monkeypatch):
    if torch.cuda.is_available():
        raise RuntimeError("the paged-cache stand-ins are for GPU-less machines only: on a GPU the kernels run")
    from cambrian_b200 import ops
    for n in ("paged_kv_append", "attn_decode_paged", "attn_decode_paged_workspace"):
        monkeypatch.setattr(ops, n, globals()[n])
