"""Timeline of the fused pass on N GPUs (torchrun): where the in-kernel exchange spends its time.
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29544 tools/pass_trace_multi.py"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import kube_throttler_b200 as kt
from kube_throttler_b200 import synth

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
snap = synth.generate("C2", seed=2 + 1000 * rank, calibrate=False)
eng = kt.Engine(snap.R, snap.L, snap.LN, device=local)
uid = [kt.Engine.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
eng.comm_init(uid[0], world, rank)
eng.upload_snapshot(snap)
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
al = torch.zeros(1, device="cuda")
s = torch.cuda.Stream(); eng.set_stream(s.cuda_stream); eng.enable_trace(True)
for it in range(5):
    with torch.cuda.stream(s):
        flush.zero_(); flush.sum(); dist.all_reduce(al)
        eng.evaluate(snap.now)
    torch.cuda.synchronize()
    rows, roles = eng.trace()
    if it < 2:
        continue
    t0 = rows[:, 2].min()
    nm, nr, nf = int(roles[0]), int(roles[1]), int(roles[2])
    rec, fin = rows[nm:nm + nr], rows[nm + nr:nm + nr + nf]
    dec = rows[:nm + nr][rows[:nm + nr, 9] > 0]  # a CTA's last match / reconcile row carries its first decide sub-tile's stamps
    us = lambda a: (a.astype(np.float64) - float(t0)) / 1e3
    med = lambda a: f"{np.median(a):.1f} (max {a.max():.1f})" if len(a) else "-"
    print(f"[rank {rank}] pass {it}: launches {eng.timing().launches} span {max(us(rows[:, 3]).max(), us(rows[:, 29]).max()):.1f} us on {int(roles[3])} CTAs | "
          f"reconcile end max {us(rec[:, 3]).max():.1f} | status: own reconcile seen {med(us(fin[:, 5]))}, totals of all ranks read {med(us(fin[:, 6]))}, "
          f"done {med(us(fin[:, 3]))} | first decide sub-tiles: sums of all ranks seen {med(us(dec[:, 11]))}, decided {med(us(dec[:, 13]))}", flush=True)
eng.close()
dist.destroy_process_group()
