"""CPU checks of 8-bit AdamW (`TrainEngine(optim="adamw_bnb_8bit")`, adam8bit.py): the two maps, the quantiser's edge
cases, the 8-bit layout, which parameters keep fp32 moments, the byte accounting, `optim` resolution, ABI argument
checks, and the engine through the CPU stand-ins (tests/adam8bit_reference.py) against a hand-written per-parameter
loop, under ZeRO-2 on two gloo ranks and with offload.  The kernels' own arithmetic is covered by
tests/test_adam8bit_gpu.py."""
import ctypes
import os
import re
import sys
from pathlib import Path

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import adam8bit_reference as R  # noqa: E402

ROOT = Path(HERE).parent
cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only; "
                                                                      "the GPU suite runs the real kernels")


# ---- format -----------------------------------------------------------------------------------------------------------
def _old_signed_map():
    """quant.dynamic_map() as it was before it took `signed`: the NF4 format's scales are coded against it."""
    data = [0.0, 1.0]
    for i in range(7):
        b = torch.linspace(0.1, 1, 2 ** i + 1, dtype=torch.float32)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (i - 6)) * means).tolist() + (-(10 ** (i - 6)) * means).tolist()
    return torch.tensor(sorted(data), dtype=torch.float32)


def _kernel_table(name):
    text = (ROOT / "cambrian_b200" / "csrc" / "adam8bit.cu").read_text()
    body = text[text.index(f"{name}[256] = {{"):]
    body = body[:body.index("};")]
    return torch.tensor([float.fromhex(x) for x in re.findall(r"(-?0x[0-9a-fp.+-]+)f", body)], dtype=torch.float32)


def test_maps():
    from cambrian_b200 import adam8bit, quant
    s, u = adam8bit.signed_map(), adam8bit.unsigned_map()
    for m in (s, u):
        assert m.numel() == 256 and bool((m[1:] > m[:-1]).all()) and m[-1] == 1.0 and (m == 0).sum() == 1
    assert torch.equal(quant.dynamic_map().view(torch.int32), _old_signed_map().view(torch.int32))
    assert torch.equal(s.view(torch.int32), _old_signed_map().view(torch.int32))
    assert u[0] == 0 and bool((u >= 0).all())
    assert torch.equal(s, R.SMAP) and torch.equal(u, R.UMAP)
    # the kernel's constant tables are these maps, bit for bit
    assert torch.equal(_kernel_table("c_a8_signed").view(torch.int32), s.view(torch.int32))
    assert torch.equal(_kernel_table("c_a8_unsigned").view(torch.int32), u.view(torch.int32))


def test_quantiser_edge_cases():
    for qmap, zero in ((R.SMAP, R.SZERO), (R.UMAP, 0)):
        # all-zero block (and a partial last block of zeros)
        q, a = R.quantize(torch.zeros(300), qmap, zero)
        assert (q == zero).all() and (a == 0).all() and a.numel() == 2
        # exact map entries round-trip, +-absmax hits the ends
        x = qmap.clone()
        q, a = R.quantize(x, qmap, zero)
        assert a.item() == 1.0 and torch.equal(q.long(), torch.arange(256))
        assert torch.equal(R.dequantize(q, a, qmap), x)
        x = qmap * 3.0                                   # exact in fp32: scaling by 3 and by 1/3 ... checked via codes
        q, a = R.quantize(x, qmap, zero)
        assert a.item() == 3.0 and q[-1] == 255
        # ties go to the larger entry; one step off the midpoint goes to the nearer one
        for j in (10, 128, 200):
            mid = (qmap[j] + qmap[j + 1]) / 2
            if (qmap[j + 1] - mid) == (mid - qmap[j]):
                q, _ = R.quantize(torch.tensor([1.0] + [mid.item()] * 7), qmap, zero)
                assert q[1] == j + 1
            below = torch.nextafter(mid, torch.tensor(-1.0))
            q, _ = R.quantize(torch.tensor([1.0] + [below.item()] * 7), qmap, zero)
            assert q[1] == j
    # signed: -absmax
    q, a = R.quantize(torch.tensor([-2.0, 1.0, 0.0, 0.5] * 2), R.SMAP, R.SZERO)
    assert q[0] == 0 and q[2] == R.SZERO and a.item() == 2.0
    # partial last block: its own absmax
    x = torch.cat([torch.full((256,), 4.0), torch.full((40,), 0.5)])
    q, a = R.quantize(x, R.UMAP, 0)
    assert a.tolist() == [4.0, 0.5] and (q == 255).all()


# ---- engine host logic --------------------------------------------------------------------------------------------------
class _Toy(torch.nn.Module):
    """An embedding, a large and a small linear, a norm: every state-format rule is exercised."""

    def __init__(self, dim=96, vocab=100):
        super().__init__()
        torch.manual_seed(0)
        self.embed = torch.nn.Embedding(vocab, dim)
        self.big = torch.nn.Linear(dim, 3 * dim + 8)
        self.small = torch.nn.Linear(dim, 24, bias=False)
        self.norm = torch.nn.LayerNorm(dim)
        self.head = torch.nn.Linear(dim, vocab, bias=False)
        self.to(torch.bfloat16)

    def forward(self, ids):
        h = self.embed(ids)
        h = h + self.big(h)[..., :h.shape[-1]] + 0.1 * self.small(h).sum(-1, keepdim=True)
        return self.head(self.norm(h)).float().logsumexp(-1).mean()


def _engine(model=None, **kw):
    from cambrian_b200.engine import TrainEngine
    return TrainEngine(model or _Toy(), lr=1e-2, weight_decay=0.1, **kw)


@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("zero_stage", [0, 2])
def test_8bit_layout_is_block_aligned(monkeypatch, world, zero_stage):
    from cambrian_b200 import engine as E
    monkeypatch.setattr(E.dist, "is_initialized", lambda: world > 1)
    monkeypatch.setattr(E.dist, "get_world_size", lambda pg=None: world)
    monkeypatch.setattr(E.dist, "get_rank", lambda pg=None: world - 1)
    eng = _engine(zero_stage=zero_stage, bucket_mb=0.05, optim="adamw_bnb_8bit")
    assert len(eng.buckets) >= 2
    assert all(o % 256 == 0 for o in eng.offsets)
    for s, e, _ in eng.buckets:
        assert s % 256 == 0 and (e - s) % (256 * world) == 0
        if zero_stage == 2:
            assert ((e - s) // world) % 256 == 0
    for b in range(len(eng.buckets)):
        for (lo, hi, _, f32, mo) in eng._segments(b, ()):
            if not f32:
                assert lo % 256 == 0 and (hi - lo) % 256 == 0 and mo % 256 == 0
    # the default layout follows the fp32-moment rule: each parameter 8-aligned right after the previous one, a bucket
    # closed once it reaches bucket_mb and padded to 8 * world elements under ZeRO-2 (to 8 otherwise)
    d = _engine(zero_stage=zero_stage, bucket_mb=0.05)
    assert len(d.buckets) >= 2
    limit = int(0.05 * 1024 * 1024 / 2)
    align = 8 * world if zero_stage == 2 else 8
    offs, total, start, buckets, cur = [], 0, 0, [], []
    for i, p in enumerate(d.params):
        offs.append(total)
        total += -(-p.numel() // 8) * 8
        cur.append(i)
        if total - start >= limit:
            total = -(-(total - start) // align) * align + start
            buckets.append((start, total, cur))
            start, cur = total, []
    if cur:
        total = -(-(total - start) // align) * align + start
        buckets.append((start, total, cur))
    assert d.offsets == offs and d.buckets == buckets and d.total == total
    assert d.exp_avg.numel() == (d.shard if zero_stage == 2 else d.total) and not hasattr(d, "exp_avg_code")


def test_which_parameters_keep_fp32_moments():
    eng = _engine(optim="adamw_bnb_8bit")
    f32 = dict(zip(eng.names, eng._fp32m))
    assert f32["embed.weight"] and f32["small.weight"] and f32["big.bias"] and f32["norm.weight"]
    assert not f32["big.weight"] and not f32["head.weight"]
    n32 = sum(-(-p.numel() // 8) * 8 for p, f in zip(eng.params, eng._fp32m) if f)
    n8 = sum(-(-p.numel() // 256) * 256 for p, f in zip(eng.params, eng._fp32m) if not f)
    assert (eng._n32, eng._n8) == (n32, n8)
    assert eng.exp_avg.numel() == n32 and eng.exp_avg_code.numel() == n8 and eng.exp_avg_absmax.numel() == n8 // 256


def test_state_bytes_formula():
    eng = _engine(optim="adamw_8bit")
    opt = 4 * eng.master.numel() + 8 * eng._n32 + 2 * eng._n8 + 8 * (eng._n8 // 256)
    assert eng.state_bytes() == 4 * eng.total + opt and eng.host_state_bytes() == 0
    d = _engine()
    assert d.state_bytes() == 16 * d.total


def test_optim_resolution_and_refusals():
    from cambrian_b200 import adam8bit
    assert adam8bit.resolve_optim("adamw_torch") is False
    assert adam8bit.resolve_optim("adamw_bnb_8bit") is True and adam8bit.resolve_optim("adamw_8bit") is True
    with pytest.raises(NotImplementedError, match="offload_optimizer=True"):
        _engine(optim="paged_adamw_8bit")
    for bad in ("adamw_hf", "sgd", "adafactor", "ADAMW_BNB_8BIT"):
        with pytest.raises(ValueError, match="optim"):
            _engine(optim=bad)
    assert _engine().optim == "adamw_torch" and not _engine().eight_bit


def _call(lib, fn, ptrs, n, step=1, last=0):
    F = ctypes.c_float
    return getattr(lib, fn)(*ptrs, n, F(1e-3), F(0.9), F(0.999), F(1e-8), F(0.0), step, F(1.0), None, last, None)


@pytest.mark.parametrize("fn", ["cb_adamw8", "cb_adamw8_host"])
def test_abi_rejects_bad_arguments_without_gpu(lib, fn):
    op = fn[3:].encode()
    one = ctypes.c_void_p(16)
    assert _call(lib, fn, [one] * 7, 12) == 1 and b"multiple of 8" in lib.cb_last_error()
    assert _call(lib, fn, [one] * 7, -8) == 1 and b"multiple of 8" in lib.cb_last_error()
    assert _call(lib, fn, [one] * 7, 8, step=0) == 1 and b"step" in lib.cb_last_error()
    names = (b"p", b"qm", b"qv", b"sm", b"sv", b"g", b"p16")
    aligns = (16, 8, 8, 4, 4, 16, 16)
    for i, (name, al) in enumerate(zip(names, aligns)):
        args = [one] * 7
        args[i] = None
        assert _call(lib, fn, args, 8) == 1 and lib.cb_last_error() == op + b": " + name + b" is null"
        args[i] = ctypes.c_void_p(16 + al // 2)
        assert _call(lib, fn, args, 8) == 1
        assert lib.cb_last_error() == op + b": " + name + b" must be %d-byte aligned" % al
    if fn == "cb_adamw8_host":
        assert _call(lib, fn, [one] * 7, 8, last=-1) == 1 and b"ctas" in lib.cb_last_error()
    assert _call(lib, fn, [None] * 7, 0) == 0


def _batches(steps, vocab=100):
    g = torch.Generator().manual_seed(5)
    return [torch.randint(0, vocab, (4, 16), generator=g) for _ in range(steps)]


def _train(eng, model, steps=4):
    losses = []
    for ids in _batches(steps):
        eng.zero_grad()
        loss = model(ids)
        loss.backward()
        eng.step()
        losses.append(float(loss.detach()))
    return losses


def _hand_loop(steps, clip=None):
    """A per-parameter 8-bit AdamW loop written from adam8bit.py's rules over the same gradients (plain autograd)."""
    from cambrian_b200 import adam8bit
    model = _Toy()
    emb = adam8bit.embedding_params(model)
    norm = {id(p) for p in model.norm.parameters()}
    state = {}
    for n, p in model.named_parameters():
        k = -(-p.numel() // 8) * 8
        master = torch.zeros(k)
        master[:p.numel()] = p.detach().float().reshape(-1)
        if adam8bit.fp32_moments(p, emb):
            state[n] = ("f32", master, torch.zeros(k), torch.zeros(k))
        else:
            k = -(-p.numel() // 256) * 256
            master = torch.cat([master, torch.zeros(k - master.numel())])
            state[n] = ("q", master, torch.full((k,), R.SZERO, dtype=torch.uint8), torch.zeros(k, dtype=torch.uint8),
                        torch.zeros(k // 256), torch.zeros(k // 256))
    import ops_emulation
    losses = []
    for t, ids in enumerate(_batches(steps), 1):
        model.zero_grad()
        loss = model(ids)
        loss.backward()
        losses.append(float(loss.detach()))
        grads = {n: p.grad.detach().reshape(-1) for n, p in model.named_parameters()}
        coef = None
        if clip is not None:
            ss = sum(float(g.float().pow(2).sum()) for g in grads.values())
            coef = torch.tensor([min(1.0, clip / (ss ** 0.5 + 1e-6)), ss ** 0.5])
        for n, p in model.named_parameters():
            st = state[n]
            k = st[1].numel()
            g16 = torch.zeros(k, dtype=torch.bfloat16)
            g16[:p.numel()] = grads[n]
            p16 = torch.empty(k, dtype=torch.bfloat16)
            wd = 0.0 if (id(p) in norm or "bias" in n) else 0.1
            if st[0] == "f32":
                ops_emulation.adamw(st[1], st[2], st[3], g16, p16, 1e-2, 0.9, 0.999, 1e-8, wd, t, clip_coef=coef)
            else:
                R.adamw8(st[1], st[2], st[3], st[4], st[5], g16, p16, 1e-2, 0.9, 0.999, 1e-8, wd, t, clip_coef=coef)
            p.data.copy_(p16[:p.numel()].view(p.shape))
    return losses, {n: s[1][:p.numel()] for (n, s), p in zip(state.items(), model.parameters())}


@cpu_only
@pytest.mark.parametrize("clip", [None, 0.5])
def test_engine_equals_hand_written_8bit_loop(monkeypatch, clip):
    R.install(monkeypatch)
    model = _Toy()
    eng = _engine(model, bucket_mb=0.05, optim="adamw_bnb_8bit", max_grad_norm=clip)
    losses = _train(eng, model)
    ref_losses, masters = _hand_loop(4, clip)
    assert len(eng.buckets) >= 2
    assert losses == ref_losses
    for i, n in enumerate(eng.names):
        o, k = eng.offsets[i], eng.params[i].numel()
        if clip is None:
            assert torch.equal(eng.master[o:o + k], masters[n]), n
        else:       # the engine sums squares per bucket: the clip coefficient may differ in the last bits
            torch.testing.assert_close(eng.master[o:o + k], masters[n], rtol=1e-5, atol=1e-6)


@cpu_only
def test_offloaded_8bit_engine_equals_device_state(monkeypatch):
    R.install(monkeypatch)
    runs = []
    for offload in (False, True):
        model = _Toy()
        eng = _engine(model, bucket_mb=0.05, optim="adamw_bnb_8bit", max_grad_norm=0.5, offload_optimizer=offload)
        runs.append((_train(eng, model), eng))
    (l0, e0), (l1, e1) = runs
    assert l0 == l1
    for name in ("flat_p", "master", "exp_avg", "exp_avg_sq", "exp_avg_code", "exp_avg_sq_code", "exp_avg_absmax",
                 "exp_avg_sq_absmax"):
        assert torch.equal(getattr(e0, name), getattr(e1, name)), name
    assert e1.state_bytes() == 4 * e1.total and e1.host_state_bytes() == e0.state_bytes() - 4 * e0.total
    e1.close()


@cpu_only
def test_8bit_losses_track_32bit_on_the_stand_in(monkeypatch):
    """30 steps of the toy model through the stand-ins, 8-bit against fp32 moments: max |difference| / first loss, 0.0023
    measured, held to 0.01.  (The GPU suite holds the tiny Cambrian model to its own bound.)"""
    R.install(monkeypatch)
    out = {}
    for optim in ("adamw_torch", "adamw_bnb_8bit"):
        model = _Toy()
        eng = _engine(model, optim=optim)
        out[optim] = _train(eng, model, steps=30)
    worst = max(abs(a - b) for a, b in zip(out["adamw_bnb_8bit"], out["adamw_torch"])) / out["adamw_torch"][0]
    print(f"worst loss difference over 30 steps / first loss: {worst:.4f}")
    assert worst <= 0.01


def _zero2_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        R.install()
        alone = [dist.new_group([r]) for r in range(world)]        # a one-rank group: the single-process reference
        out = []
        for zero_stage, pg in ((0, alone[rank]), (2, None), (0, None)):
            model = _Toy()
            eng = _engine(model, bucket_mb=0.05, optim="adamw_bnb_8bit", zero_stage=zero_stage, process_group=pg)
            assert eng.world == (1 if pg is not None else world)
            # every rank sees the same batches: the averaged gradient equals one process's
            losses = _train(eng, model)
            out.append((losses, {n: eng.flat_p[o:o + p.numel()].float().numpy()
                                 for n, o, p in zip(eng.names, eng.offsets, eng.params)}))
        q.put((rank, out, None))
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, None, traceback.format_exc()[-2000:]))
    finally:
        dist.destroy_process_group()


@cpu_only
def test_zero2_two_ranks_gloo_equals_one_process():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 37500 + os.getpid() % 2000
    procs = [ctx.Process(target=_zero2_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in procs), key=lambda r: r[0])
    for p in procs:
        p.join(60)
    assert all(r[2] is None for r in res), [r[2] for r in res]
    for rank, ((single, ref), *runs), _ in res:
        for what, (losses, params) in zip(("zero2", "ddp"), runs):
            assert losses == single, (rank, what)
            for n in ref:
                assert (params[n] == ref[n]).all(), (rank, what, n)
