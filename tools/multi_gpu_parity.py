"""Multi-GPU parity: one process per GPU (torchrun), row-sharded snapshot, ONE NCCL all-reduce per pass.
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/multi_gpu_parity.py [C3] [m n p [arrival]]
"arrival": the pod rows in arrival order, which every rank lays out by namespace (kt_debug_set_row_order) for its own shard.
Rank 0 compares the stacked per-rank results with the oracle's evaluation of the WHOLE snapshot, bit for bit, and every
rank checks that its per-throttle results equal rank 0's (they come out of the same all-reduced partials)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

import kube_throttler_b200 as kt
from kube_throttler_b200 import abi, shard, synth

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
cfg = sys.argv[1] if len(sys.argv) > 1 else "C3"
kw = dict(m=int(sys.argv[2]), n=int(sys.argv[3]), p=int(sys.argv[4])) if len(sys.argv) > 4 else dict(m=1000, n=20011, p=2003)
arrival = len(sys.argv) > 5 and sys.argv[5] == "arrival"
full = synth.generate(cfg, **kw, sort_by_namespace=not arrival)
mine = shard.shard_snapshot(full, rank, world)
eng = kt.Engine(full.R, full.L, full.LN, device=local)
if arrival:
    for kind in (abi.PODS_RUNNING, abi.PODS_PENDING):
        eng.set_row_order(kind, abi.ROW_ORDER_BY_NAMESPACE)
uid = [kt.Engine.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
eng.comm_init(uid[0], world, rank)
eng.upload_snapshot(mine)
assert not arrival or all(eng.row_order(kind)[0] for kind in (abi.PODS_RUNNING, abi.PODS_PENDING))
results = []
for flags in (abi.EVAL_FRESH_STATUS, abi.EVAL_ON_EQUAL):
    eng.evaluate(full.now, flags)
    results.append(eng.download())
eng.evaluate(full.now)  # a second pass over the same state: the partial-sum buffer was consumed and re-zeroed
again = eng.download()
eng.close()
gathered = [None] * world
dist.gather_object((results, again), gathered if rank == 0 else None, dst=0)
ok = True
if rank == 0:
    from oracle import ko  # the checker

    for i, flags in enumerate((abi.EVAL_FRESH_STATUS, abi.EVAL_ON_EQUAL)):
        parts = [g[0][i] for g in gathered]
        got = shard.concat_results(parts)
        want = ko.columnar_evaluate(full, flags, words_per_row=got.words_per_row)
        live = ((full.thr_flags & abi.THR_RESPONSIBLE) != 0) & ((full.thr_flags & abi.THR_SELECTOR_ERROR) == 0)
        for f in ("run_bitmap", "pend_bitmap", "codes", "admit", "calc_thr", "calc_present", "calc_cnt", "override_active"):
            if not np.array_equal(getattr(got, f), getattr(want, f)):
                ok = False
                print(f"MISMATCH flags={flags} field={f}")
        for f in ("used", "used_present", "used_cnt", "throttled"):
            a, b = getattr(got, f), getattr(want, f)
            a, b = (a[:, live], b[:, live]) if a.ndim == 2 else (a[live], b[live])
            if not np.array_equal(a, b):
                ok = False
                print(f"MISMATCH flags={flags} field={f}")
        for r, part in enumerate(parts[1:], 1):  # replicated per-throttle results
            for f in ("used", "used_cnt", "used_present", "throttled", "calc_thr"):
                if not np.array_equal(getattr(part, f), getattr(parts[0], f)):
                    ok = False
                    print(f"rank {r} disagrees with rank 0 on {f}")
    first = shard.concat_results([g[0][0] for g in gathered])
    second = shard.concat_results([g[1] for g in gathered])
    for f in ("used", "used_cnt", "codes", "admit", "run_bitmap"):
        if not np.array_equal(getattr(first, f), getattr(second, f)):
            ok = False
            print(f"second pass differs on {f}")
    print(f"multi-gpu parity world={world} config={cfg} {kw} arrival={arrival}: {'OK' if ok else 'FAILED'}")
flag = torch.tensor([1 if ok else 0], device="cuda")
dist.broadcast(flag, src=0)
dist.destroy_process_group()
sys.exit(0 if int(flag.item()) == 1 else 1)
