"""Two-GPU (NCCL) tests of 8-bit Adam moments (`TrainEngine(optim="adamw_bnb_8bit")`): need >= 2 visible CUDA devices,
skipped otherwise.  ZeRO-2 (NCCL reduce_scatter_tensor into the rank's 256-aligned pieces, in-place all_gather) and the
in-switch / peer all-reduce on the symmetric gradient buffer (`collective="multimem"`, which falls back to peer
load/store without multicast) must reproduce 8-bit DDP over NCCL by tests/test_multi_gpu.py's criterion, with
rank-varying inputs, and every rank must hold the same parameters."""
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
        from helpers import rel_err, tiny_cambrian_config
        from cambrian_b200.engine import TrainEngine
        dev = f"cuda:{rank}"
        T.dev = dev
        calls = {"rs": 0, "ag": 0}
        rs0, ag0 = dist.reduce_scatter_tensor, dist.all_gather_into_tensor

        def rs(*a, **k):
            calls["rs"] += 1
            return rs0(*a, **k)

        def ag(*a, **k):
            calls["ag"] += 1
            return ag0(*a, **k)
        dist.reduce_scatter_tensor, dist.all_gather_into_tensor = rs, ag
        out, msg, ok = {}, "", True
        for name, zero, coll in (("ddp", 0, "nccl"), ("zero2", 2, "nccl"), ("multimem", 0, "multimem")):
            cfg = tiny_cambrian_config()
            cfg.fused_lm_loss = True
            model = T._build_tiny_model(cfg)          # same seed on every rank -> identical replicas
            model.train()
            eng = TrainEngine(model, lr=1e-3, bucket_mb=8.0, zero_stage=zero, max_grad_norm=0.05, collective=coll,
                              optim="adamw_bnb_8bit")
            eng.defer_param_sync = True
            ok &= eng._n8 > 0 and all((e - s) % (256 * world) == 0 for s, e, _ in eng.buckets)
            if zero == 2:
                ok &= eng.master.numel() * world == eng.total           # optimizer state really is sharded
            losses = []
            for step in range(3):
                ids, labels, attn, pos, images, masks = T._tiny_batch(cfg)
                images = [i + 0.1 * rank for i in images]
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
            out[name] = (eng.flat_p[: eng.offsets[-1] + eng.params[-1].numel()].float().cpu(), losses, eng._overlap_ok)
            t = out[name][0].to(dev)                                     # replicas agree across ranks
            lo, hi = t.clone(), t.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN)
            dist.all_reduce(hi, op=dist.ReduceOp.MAX)
            same = bool(torch.equal(lo, hi))
            ok &= same
            msg += f" {name}: replicas equal {same};"
        ok &= calls["rs"] > 0 and calls["ag"] > 0                      # the NCCL ZeRO-2 path was reached
        msg += f" rs={calls['rs']} ag={calls['ag']};"
        a = out["ddp"]
        for name in ("zero2", "multimem"):
            b = out[name]
            n = min(a[0].numel(), b[0].numel())
            e = rel_err(b[0][:n], a[0][:n])
            good = e < 2e-2 and all(abs(x - y) < 2e-2 * abs(x) for x, y in zip(a[1], b[1])) and a[2] and b[2]
            ok &= good
            msg += f" {name}-vs-ddp rel_err {e:.2e} losses {a[1]} {b[1]} overlap_ok {a[2]} {b[2]};"
        q.put((rank, bool(ok), msg))
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, False, traceback.format_exc()[-1500:]))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_8bit_zero2_and_multimem_match_8bit_ddp():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29000 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(60)
    print(res)
    assert all(r[1] for r in res), res
