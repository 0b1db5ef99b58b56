"""Push / pull bandwidth sweep over NVLink vs NCCL (BASELINE.json config 5).

    torchrun --nproc-per-node 2 tools/sweep_pushpull.py [--max-mb 1024]

Rank 0 owns the master segment; rank 1 (the worker) times
  pull  : pull_kernel copying the bf16 publish buffer (W and W^T) from the master over NVLink
  push  : push_kernel (SGD and Adam): gradient local, master tuples read + written over NVLink, bf16 publish
against
  nccl broadcast of the fp32 parameters (src=0) and nccl reduce of the fp32 gradient (dst=0).
All times are CUDA events on the launching stream of the worker rank (max over ranks for the collectives).
"""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import ParamLayout
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel import dist as D
from sparkflow_b200.parallel.device_engine import MasterState


def timeit(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def main():
    max_mb = int(sys.argv[sys.argv.index("--max-mb") + 1]) if "--max-mb" in sys.argv else 1024
    ctx = D.get_context()
    dev = torch.device("cuda", ctx.local_rank)
    torch.cuda.set_device(dev)
    C = native.cuda_ext()
    C.set_pdl(1)
    worker_rank = ctx.world - 1
    out = []
    sizes = [1 << k for k in range(10, 31) if (1 << k) <= max_mb << 20]          # fp32 parameter bytes
    for nbytes in sizes:
        n = nbytes // 4
        cols = 4096 if n >= 4096 * 32 else max(8, min(n, 256))
        rows = max(1, n // cols)
        lay = ParamLayout.build([("w/kernel", (rows, cols))])
        iters = 20 if nbytes <= (64 << 20) else 5
        rec = {"param_bytes": rows * cols * 4}
        for opt in ("gradient_descent", "adam"):
            spec = OptimizerSpec.from_tf_kwargs(opt, dict(learning_rate=1e-3))
            if ctx.is_master:
                master = MasterState(lay, spec, dev, n_mailboxes=ctx.world)
                master.load_weights([np.zeros((rows, cols), np.float32)])
                handle = master.ipc_handle()
            else:
                handle = None
            handle = D.broadcast_object(ctx, handle, 0)
            if not ctx.is_master:
                master = MasterState.from_ipc(lay, spec, dev, handle, n_mailboxes=ctx.world)
            D.barrier(ctx)
            if ctx.rank == worker_rank:
                grads = torch.full((lay.total,), 1e-3, device=dev)
                segs = torch.frombuffer(bytearray(C.pack_segs(lay.seg_rows())), dtype=torch.uint8).to(dev)
                tmap = torch.from_numpy(lay.tile_map()).to(dev)
                sync = torch.zeros(16, dtype=torch.int32, device=dev)
                loss = torch.zeros(2, device=dev)
                replica = torch.zeros(lay.shadow_total, dtype=torch.bfloat16, device=dev)
                seen = torch.zeros(1, dtype=torch.int32, device=dev)
                pargs = dict(state=native.ptr(master.state), ctrl=native.ptr(master.ctrl), shadow_dst=[native.ptr(master.shadow)],
                             grad=native.ptr(grads), loss_acc=native.ptr(loss), loss_out=native.ptr(loss) + 4, segs=native.ptr(segs),
                             tile_map=native.ptr(tmap), num_tiles=int(tmap.shape[0]), seg_rows=lay.seg_rows(), optimizer=spec.opt_id,
                             lock_mode=0, scope_sys=1, grad_scale=1.0, hyper=spec.native_hyper())
                qargs = dict(src=native.ptr(master.shadow), dst=native.ptr(replica), n_bf16=lay.shadow_total, n_f32=0,
                             ctrl=native.ptr(master.ctrl), seen_version=native.ptr(seen), lock_mode=0, scope_sys=1)
                st = native.current_stream()
                t_push = timeit(lambda: C.push(pargs, native.ptr(sync), 0, st), iters)
                rec[f"push_{opt}_s"] = t_push
                # NVLink bytes of a push: 16 B tuple read + 16 B tuple write + 2 x 2 B publish, per parameter
                rec[f"push_{opt}_nvlink_GBs"] = rows * cols * 36 / t_push / 1e9
                if opt == "adam":
                    t_pull = timeit(lambda: C.pull(qargs, native.ptr(sync) + 32, 0, st), iters)
                    rec["pull_s"] = t_pull
                    rec["pull_nvlink_GBs"] = lay.shadow_total * 2 / t_pull / 1e9
            D.barrier(ctx)
            if opt == "adam":
                # served push: the worker only streams its gradient into its mailbox (4 B / parameter over NVLink);
                # the applier on the master GPU applies it.  Back-to-back posts wait for the previous apply, so this
                # is the sustained post + apply rate of one worker.
                if ctx.is_master:
                    master.start_applier(False, scope_sys=True)
                D.barrier(ctx)
                if ctx.rank == worker_rank:
                    psync = torch.zeros(16, dtype=torch.int32, device=dev)
                    post_args = dict(grad=native.ptr(grads), mailbox=master.mailbox_ptr(ctx.rank), flags=master.flags_ptr(ctx.rank),
                                     loss_acc=native.ptr(loss), loss_out=native.ptr(loss) + 4, n=lay.total)
                    t_post = timeit(lambda: C.post(post_args, native.ptr(psync), 0, st), iters)
                    rec["served_push_s"] = t_post
                    rec["served_push_nvlink_GBs"] = rows * cols * 4 / t_post / 1e9
                    import time
                    time.sleep(0.05)
                D.barrier(ctx)
                if ctx.is_master:
                    master.stop_applier()
                D.barrier(ctx)
            torch.cuda.synchronize()
            if ctx.is_master:
                master.close()
            else:
                master.close()
            D.barrier(ctx)
        # NCCL arm: broadcast fp32 params + reduce fp32 grads
        buf = torch.zeros(rows * cols, device=dev)
        t_b = timeit(lambda: dist.broadcast(buf, src=0), iters)
        t_r = timeit(lambda: dist.reduce(buf, dst=0), iters)
        tb = max(D.all_gather_object(ctx, t_b))
        tr = max(D.all_gather_object(ctx, t_r))
        rec["nccl_broadcast_s"], rec["nccl_broadcast_GBs"] = tb, rows * cols * 4 / tb / 1e9
        rec["nccl_reduce_s"], rec["nccl_reduce_GBs"] = tr, rows * cols * 4 / tr / 1e9
        allrec = D.all_gather_object(ctx, rec)
        if ctx.is_master:
            merged = {}
            for r in allrec:
                merged.update(r)
            out.append(merged)
            print(json.dumps(merged), flush=True)
    if ctx.is_master:
        os.makedirs("bench_out", exist_ok=True)
        json.dump(out, open("bench_out/sweep_pushpull.json", "w"), indent=1)


if __name__ == "__main__":
    main()
