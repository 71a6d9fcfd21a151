"""GPU tests of the host-resident optimizer state: `ops.adamw_host` (cb_adamw_host, offload.cu) on registered host arrays
is bitwise equal to `ops.adamw` on device copies; misplaced operands are rejected before any launch; and
`TrainEngine(offload_optimizer=True)` trains bit for bit like the device-state engine in every schedule while holding
12 B per optimizer element less on the device."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_engine_gpu import _setup  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"
SWEEP_CTAS = (4, 8, 16, 32, 64, 132)


class _PointerAttributes(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int), ("device", ctypes.c_int), ("devicePointer", ctypes.c_void_p),
                ("hostPointer", ctypes.c_void_p)]


def _memory_type(t):
    """cudaPointerGetAttributes(t).type: 0 unregistered, 1 registered host, 2 device, 3 managed."""
    torch.cuda.init()
    try:
        cudart = ctypes.CDLL("libcudart.so.12")      # torch's own runtime, already loaded into the process
    except OSError:
        import glob
        import nvidia
        cudart = ctypes.CDLL(glob.glob(os.path.join(nvidia.__path__[0], "cuda_runtime", "lib", "libcudart.so.12*"))[0])
    a = _PointerAttributes()
    assert cudart.cudaPointerGetAttributes(ctypes.byref(a), ctypes.c_void_p(t.data_ptr())) == 0
    return a.type


def _registered(*ts):
    from cambrian_b200 import ops
    for t in ts:
        ops.host_register(t)
    return ts


def _unregister(*ts):
    from cambrian_b200 import ops
    torch.cuda.synchronize()
    for t in ts:
        ops.host_unregister(t)


@pytest.mark.parametrize("n", [8, 8 * 4099, 8 * (2 ** 20 + 3)])
def test_adamw_host_is_bitwise_equal_to_device_adamw(n):
    from cambrian_b200 import ops
    gen = torch.Generator(device=dev).manual_seed(n)
    p0 = torch.randn(n, device=dev, generator=gen)
    m0 = torch.randn(n, device=dev, generator=gen) * 1e-2
    v0 = torch.rand(n, device=dev, generator=gen) * 1e-4
    g = torch.randn(n, device=dev, generator=gen).bfloat16()
    hp, hm, hv = _registered(torch.empty(n), torch.empty(n), torch.empty(n))
    try:
        for clip in (False, True):
            coef = torch.tensor([0.37, 0.0], device=dev) if clip else None
            for wd in (0.0, 0.1):
                p, m, v = p0.clone(), m0.clone(), v0.clone()
                p16 = torch.empty(n, device=dev, dtype=torch.bfloat16)
                for step in (1, 2, 3, 1000):
                    ops.adamw(p, m, v, g, p16, 1e-2, 0.9, 0.999, 1e-8, wd, step, grad_scale=0.5, clip_coef=coef)
                for ctas in (0,) + SWEEP_CTAS:
                    hp.copy_(p0.cpu()), hm.copy_(m0.cpu()), hv.copy_(v0.cpu())
                    h16 = torch.full((n,), 7.0, device=dev, dtype=torch.bfloat16)
                    for step in (1, 2, 3, 1000):
                        ops.adamw_host(hp, hm, hv, g, h16, 1e-2, 0.9, 0.999, 1e-8, wd, step, grad_scale=0.5, clip_coef=coef,
                                       ctas=ctas)
                    torch.cuda.synchronize()
                    what = f"n={n} clip={clip} wd={wd} ctas={ctas}"
                    assert torch.equal(hp, p.cpu()), what
                    assert torch.equal(hm, m.cpu()), what
                    assert torch.equal(hv, v.cpu()), what
                    assert torch.equal(h16, p16), what
    finally:
        _unregister(hp, hm, hv)


def test_adamw_host_rejects_misplaced_operands_before_launching():
    from cambrian_b200 import _lib, ops
    n = 8 * 1024
    g = torch.randn(n, device=dev).bfloat16()
    p16 = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    hp, hm, hv = _registered(torch.ones(n), torch.ones(n), torch.ones(n))
    pageable = torch.ones(n)
    try:
        torch.cuda.synchronize()
        lib = _lib.load()
        cases = [((hp, torch.ones(n, device=dev), hv, g, p16), "m must be host memory registered", "got device memory"),
                 ((pageable, hm, hv, g, p16), "p must be host memory registered", "got unregistered"),
                 ((hp, hm, hv, torch.ones(n).bfloat16(), p16), "g must be device memory", "got unregistered"),
                 ((hp, hm, hv, _registered(torch.ones(n).bfloat16())[0], p16), "g must be device memory",
                  "got registered host memory"),
                 ((hp, hm, hv, g, torch.zeros(n).bfloat16()), "p16 must be device memory", "got unregistered")]
        for args, what, kind in cases:
            before = lib.cb_launch_count()
            with pytest.raises(ValueError, match=what) as ei:
                ops.adamw_host(*args, 1e-2, 0.9, 0.999, 1e-8, 0.0, 1)
            assert kind in str(ei.value)
            assert lib.cb_launch_count() == before, what          # nothing was launched
        _unregister(cases[3][0][3])
        torch.cuda.synchronize()
        assert torch.equal(hp, torch.ones(n)) and torch.equal(pageable, torch.ones(n)) and not p16.any()
        # a healthy call afterwards: the rejected ones left no CUDA error behind
        ops.adamw_host(hp, hm, hv, g, p16, 1e-2, 0.9, 0.999, 1e-8, 0.0, 1)
        torch.cuda.synchronize()
        assert p16.any()
    finally:
        _unregister(hp, hm, hv)


SCHEDULES = [(True, False), (False, False), (True, True)]      # (overlap, defer_param_sync): overlapped, serial, deferred


def _train(offload, overlap, defer, bg, clip, bucket_mb=8.0):
    from cambrian_b200.engine import TrainEngine
    cfg, model, batch = _setup()
    eng = TrainEngine(model, lr=1e-3, bucket_mb=bucket_mb, overlap=overlap, max_grad_norm=clip, background_optimizer=bg,
                      offload_optimizer=offload)
    eng.defer_param_sync = defer
    losses = []
    for _ in range(3):
        eng.zero_grad()
        loss = model(**batch).loss
        loss.backward()
        eng.step()
        losses.append(float(loss.detach()))
    eng.wait_for_params()
    torch.cuda.synchronize()
    return eng, losses


@pytest.mark.parametrize("clip", [None, 0.05])
@pytest.mark.parametrize("bg", [True, False])
@pytest.mark.parametrize("overlap,defer", SCHEDULES)
def test_offloaded_engine_is_bitwise_equal_in_every_schedule(overlap, defer, bg, clip):
    ref, ref_losses = _train(False, overlap, defer, bg, clip)
    eng, losses = _train(True, overlap, defer, bg, clip)
    try:
        assert len(eng.buckets) > 3
        assert _memory_type(eng.master) == 1 and _memory_type(eng.exp_avg) == 1 and _memory_type(eng.exp_avg_sq) == 1
        assert eng._opt_stream is not None                  # the update still runs on the optimizer's side stream
        assert losses == ref_losses
        assert torch.equal(eng.flat_p, ref.flat_p)
        for name in ("master", "exp_avg", "exp_avg_sq"):
            assert torch.equal(getattr(eng, name), getattr(ref, name).cpu()), name
    finally:
        eng.close()


def test_offload_memory_accounting_and_lifetime():
    from cambrian_b200.engine import TrainEngine
    torch.cuda.synchronize()
    used = {}
    engines = {}
    for offload in (False, True):
        cfg, model, batch = _setup()
        # the engine moves every parameter into its flat buffer and frees the old storage; keeping that storage alive until
        # the engine is measured leaves the count to the engine's own allocations (the blocks the freed parameters held
        # depend on what the caching allocator had cached when the model was built)
        old_storage = [p.data for p in model.parameters()]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        eng = TrainEngine(model, lr=1e-3, bucket_mb=0.5, offload_optimizer=offload)
        torch.cuda.synchronize()
        used[offload] = (torch.cuda.memory_allocated() - before, torch.cuda.max_memory_allocated() - before)
        engines[offload] = (eng, model, batch)
        del old_storage
    ref, eng = engines[False][0], engines[True][0]
    n_state = eng.master.numel()
    assert n_state == eng.total and len(eng.buckets) > 3
    # the device holds 12 B per optimizer element less, within the caching allocator's granularity (a large block is not
    # split when less than 1 MB would remain)
    assert 0 <= (used[False][0] - used[True][0]) - 12 * n_state <= 3 * 2 ** 20
    assert eng.state_bytes() == 4 * eng.total and ref.state_bytes() == 16 * eng.total
    # construction never held more than the engine's device buffers plus one bucket's fp32 scratch
    buffers = sum(t.numel() * t.element_size() for t in (eng.flat_p, eng.flat_g, eng._sumsq, eng._coef))
    scratch = 4 * max(e - s for s, e, _ in eng.buckets)
    assert scratch * 8 < 12 * n_state
    assert used[True][1] <= buffers + scratch + 6 * 2 ** 20, (used[True][1], buffers, scratch)
    registered = [t for t in (eng.master, eng.exp_avg, eng.exp_avg_sq) if _memory_type(t) == 1]
    assert eng.host_state_bytes() == sum(t.numel() * 4 for t in registered) == 12 * n_state
    assert ref.host_state_bytes() == 0
    # lifetime: close() unregisters (idempotently) and the engine refuses to step
    _, model, batch = engines[True]
    eng.zero_grad()
    model(**batch).loss.backward()
    eng.step()
    state = (eng.master, eng.exp_avg, eng.exp_avg_sq)
    eng.close()
    assert [_memory_type(t) for t in state] == [0, 0, 0]
    eng.close()
    with pytest.raises(RuntimeError, match="close"):
        eng.step()
