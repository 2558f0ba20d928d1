"""Which reconcile tiles are slow?  Correlates the in-kernel trace with each tile's namespace / word count / match count."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import kube_throttler_b200 as kt
from kube_throttler_b200 import synth
print("gen", flush=True); snap = synth.generate("C2")
eng = kt.Engine(snap.R, snap.L, snap.LN)
eng.upload_snapshot(snap)
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
s = torch.cuda.Stream(); eng.set_stream(s.cuda_stream); eng.enable_trace(True)
for it in range(3):
    with torch.cuda.stream(s):
        flush.zero_(); flush.sum(); eng.evaluate(snap.now)
    torch.cuda.synchronize(); print("pass", it, flush=True)
print("passes done", flush=True); rows, roles = eng.trace(); print("trace ok", flush=True)
res = eng.download(); print("download ok", flush=True)
t0 = rows[:, 2].min()
nm, nr = int(roles[0]), int(roles[1])
rec = rows[nm:nm + nr]
dur = (rec[:, 3] - rec[:, 2]) / 1e3
end = (rec[:, 3] - t0) / 1e3
ns = snap.running.ns_id
bm = res.run_bitmap
matches = np.array([int(np.unpackbits(bm[i * 128:(i + 1) * 128].view(np.uint8)).sum()) for i in range(nr)])
nns = np.array([len(set(ns[i * 128:(i + 1) * 128])) for i in range(nr)])
words = np.array([int((bm[i * 128:(i + 1) * 128] != 0).any(axis=0).sum()) for i in range(nr)])
sm = rec[:, 1].astype(int)
per_sm = np.bincount(sm, minlength=132)
print("corr(dur, matches) %.2f  corr(dur, words) %.2f  corr(dur, ctas_on_sm) %.2f  corr(end, start) %.2f" % (
    np.corrcoef(dur, matches)[0, 1], np.corrcoef(dur, words)[0, 1], np.corrcoef(dur, per_sm[sm])[0, 1], np.corrcoef(end, (rec[:, 2] - t0) / 1e3)[0, 1]))
order = np.argsort(-end)[:12]
for i in order:
    print(f"tile {i:4d} sm {sm[i]:3d} (ctas on sm {per_sm[sm[i]]}) start {(rec[i,2]-t0)/1e3:5.1f} end {end[i]:5.1f} dur {dur[i]:5.1f} matches {matches[i]:5d} words {words[i]} ns {nns[i]}")
print("dur percentiles", np.percentile(dur, [5, 25, 50, 75, 95, 100]).round(1), "end percentiles", np.percentile(end, [5, 25, 50, 75, 95, 100]).round(1))
allsm = np.bincount(rows[:, 1].astype(int), minlength=132)
print("CTAs per SM (all roles): min %d max %d" % (allsm.min(), allsm.max()))
for lo, hi in ((0, 200), (200, 500), (500, 900), (900, 2000), (2000, 100000)):
    m = (matches >= lo) & (matches < hi)
    if m.any(): print(f"matches [{lo},{hi}): n={m.sum():4d} median dur {np.median(dur[m]):5.1f} median end {np.median(end[m]):5.1f}")
eng.close()
