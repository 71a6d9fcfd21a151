"""CPU checks of the host-resident optimizer state (`TrainEngine(offload_optimizer=True)`, `cb_adamw_host`): the entry
point rejects bad arguments before any CUDA call, and the engine's offload path (host allocation, bucket-by-bucket master
fill, the same slices / segments / step / clip coefficient handed to the update) trains exactly like the device path,
alone and on two gloo ranks under ZeRO-2.  The kernels are replaced by plain-torch stand-ins (tests/ops_emulation.py, and
`adamw_host` below); the kernel's own arithmetic is covered by tests/test_offload_gpu.py."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ops_emulation  # noqa: E402

F = ctypes.c_float


def _call(lib, p, m, v, g, p16, n, step=1, ctas=0):
    return lib.cb_adamw_host(p, m, v, g, p16, n, F(1e-3), F(0.9), F(0.999), F(1e-8), F(0.0), step, F(1.0), None, ctas, None)


def test_adamw_host_rejects_bad_arguments_without_gpu(lib):
    one = ctypes.c_void_p(16)                      # non-null, 16-byte aligned dummy pointer (never dereferenced)
    assert _call(lib, one, one, one, one, one, 12) == 1 and b"multiple of 8" in lib.cb_last_error()
    assert _call(lib, one, one, one, one, one, -8) == 1 and b"multiple of 8" in lib.cb_last_error()
    assert _call(lib, one, one, one, one, one, 8, step=0) == 1 and b"step" in lib.cb_last_error()
    assert _call(lib, one, one, one, one, one, 8, ctas=-1) == 1 and b"ctas" in lib.cb_last_error()
    for i, name in enumerate((b"p", b"m", b"v", b"g", b"p16")):
        args = [one] * 5
        args[i] = None
        assert _call(lib, *args, 8) == 1 and lib.cb_last_error() == b"adamw_host: " + name + b" is null"
        args[i] = ctypes.c_void_p(24)
        assert _call(lib, *args, 8) == 1 and lib.cb_last_error() == b"adamw_host: " + name + b" must be 16-byte aligned"
    assert _call(lib, None, None, None, None, None, 0) == 0      # an empty range is a no-op, as for cb_adamw_ex


def adamw_host(p32, m, v, g16, p16, lr, beta1, beta2, eps, wd, step, grad_scale=1.0, clip_coef=None, ctas=0):
    """Stand-in for the offload kernel: the arithmetic of adamw_kernel (the kernel is bitwise equal to it on the GPU); the
    state must be CPU tensors, as the engine allocates them."""
    assert not p32.is_cuda and not m.is_cuda and not v.is_cuda
    ops_emulation.adamw(p32, m, v, g16, p16, lr, beta1, beta2, eps, wd, step, grad_scale=grad_scale, clip_coef=clip_coef)


def _install(monkeypatch=None):
    ops_emulation.install(monkeypatch)
    from cambrian_b200 import ops
    (monkeypatch or ops_emulation._Setter).setattr(ops, "adamw_host", adamw_host)


def _sampler():
    from cambrian_b200.model.vision_sampler import VisionTokenSampler
    torch.manual_seed(0)
    return VisionTokenSampler(256, 1024, [1024] * 2, [1, 2], 1024, 1).to(torch.bfloat16)


def _train(m, eng, rank=0, steps=3):
    B, qs = 2, 2
    losses = []
    for step in range(steps):
        g = torch.Generator().manual_seed(1000 * step + rank)
        q_ = torch.randn(B * qs * qs, 1, 256, generator=g).bfloat16()
        c_ = torch.randn(B * qs * qs, 1, 1024, generator=g).bfloat16()
        feats = [torch.randn(B, (r * qs) ** 2, 1024, generator=g).bfloat16() for r in (1, 2)]
        eng.zero_grad()
        loss = m(q_, c_, *feats, natural_layout=(B, qs)).float().pow(2).mean()
        loss.backward()
        eng.step()
        losses.append(float(loss.detach()))
    return losses


def _state(eng):
    return [eng.flat_p.clone(), eng.master.clone(), eng.exp_avg.clone(), eng.exp_avg_sq.clone()]


cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="kernel stand-ins are for GPU-less machines only; "
                                                                      "the GPU suite runs the real kernel")


@cpu_only
@pytest.mark.parametrize("clip,schedule", [(None, False), (0.05, False), (0.05, True)])
def test_offloaded_engine_equals_device_engine(monkeypatch, clip, schedule):
    from cambrian_b200.engine import TrainEngine, cosine_schedule_with_warmup
    _install(monkeypatch)
    runs = []
    for offload in (False, True):
        m = _sampler()
        eng = TrainEngine(m, lr=1e-3, weight_decay=0.1, bucket_mb=2.0, max_grad_norm=clip, offload_optimizer=offload,
                          lr_lambda=cosine_schedule_with_warmup(1, 3) if schedule else None)
        assert len(eng.buckets) >= 3 and not eng.master.is_cuda and eng.master.dtype == torch.float32
        runs.append((_train(m, eng), _state(eng), eng))
    (l0, s0, e0), (l1, s1, e1) = runs
    assert l0 == l1
    for name, a, b in zip(("flat_p", "master", "exp_avg", "exp_avg_sq"), s0, s1):
        assert torch.equal(a, b), name
    assert e1.state_bytes() == e1.total * 4 and e0.state_bytes() == e1.total * 16
    assert e1.host_state_bytes() == 12 * e1.total and e0.host_state_bytes() == 0
    e1.close()
    e1.close()                                     # idempotent
    with pytest.raises(RuntimeError, match="close"):
        e1.step()


def _zero2_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // (2 * world)))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _install()
        from cambrian_b200.engine import TrainEngine
        out = []
        for offload in (False, True):
            m = _sampler()
            eng = TrainEngine(m, lr=1e-3, bucket_mb=2.0, zero_stage=2, max_grad_norm=0.05, offload_optimizer=offload)
            losses = _train(m, eng, rank)
            out.append((losses, [t.float().numpy() for t in _state(eng)], eng.master.numel() * world == eng.total))
        q.put((rank, out, None))
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, None, traceback.format_exc()[-2000:]))
    finally:
        dist.destroy_process_group()


@cpu_only
def test_offloaded_zero2_two_ranks_gloo_equals_device_state():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 36500 + os.getpid() % 2000
    procs = [ctx.Process(target=_zero2_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in procs), key=lambda r: r[0])
    for p in procs:
        p.join(60)
    assert all(r[2] is None for r in res), [r[2] for r in res]
    for rank, ((l0, s0, sharded0), (l1, s1, sharded1)), _ in res:
        assert sharded0 and sharded1
        assert l0 == l1, rank
        for name, a, b in zip(("flat_p", "master", "exp_avg", "exp_avg_sq"), s0, s1):
            assert (a == b).all(), (rank, name)
