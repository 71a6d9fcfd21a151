"""Two-GPU (NCCL) test of the host-resident optimizer state: ZeRO-2 with `offload_optimizer=True` (every rank's pieces of
the fp32 master and moments in registered host memory) trains bit for bit like ZeRO-2 with device state.  Needs >= 2
visible CUDA devices, skipped otherwise."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import sys
    import torch.distributed as dist
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, here)
    sys.path.insert(0, os.path.dirname(here))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import test_modules_gpu as T
        from helpers import tiny_cambrian_config
        from cambrian_b200.engine import TrainEngine
        dev = f"cuda:{rank}"
        T.dev = dev
        out = {}
        for offload in (False, True):
            cfg = tiny_cambrian_config()
            cfg.fused_lm_loss = True
            model = T._build_tiny_model(cfg)          # same seed on every rank -> identical replicas
            model.train()
            eng = TrainEngine(model, lr=1e-3, bucket_mb=8.0, zero_stage=2, max_grad_norm=0.05, offload_optimizer=offload)
            eng.defer_param_sync = True
            losses = []
            for step in range(3):
                ids, labels, attn, pos, images, masks = T._tiny_batch(cfg)
                images = [i + 0.1 * rank for i in images]                  # rank-dependent data
                batch = dict(input_ids=ids.to(dev), labels=labels.to(dev), attention_mask=attn.to(dev),
                             position_ids=pos.to(dev), images=[i.to(dev).bfloat16() for i in images],
                             image_aux_attention_masks_list=[m.to(dev) for m in masks])
                eng.zero_grad()
                loss = model(**batch).loss
                loss.backward()
                eng.step()
                losses.append(float(loss.detach()))
            eng.wait_for_params()
            torch.cuda.synchronize()
            out[offload] = (losses, eng.flat_p.cpu(), eng.master.cpu(), eng.exp_avg.cpu(), eng.exp_avg_sq.cpu(),
                            eng.master.numel() * world == eng.total, eng.master.is_cuda)
            eng.close()
        a, b = out[False], out[True]
        ok = a[0] == b[0] and all(torch.equal(x, y) for x, y in zip(a[1:5], b[1:5])) and a[5] and b[5]
        ok &= a[6] and not b[6]
        q.put((rank, bool(ok), f"losses {a[0]} {b[0]}"))
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, False, traceback.format_exc()[-1500:]))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_offloaded_zero2_nccl_is_bitwise_equal_to_device_state():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 25000 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(60)
    assert all(r[1] for r in res), res
