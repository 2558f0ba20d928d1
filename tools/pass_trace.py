"""Per-role timeline of the fused pass (k_pass) from the in-kernel trace: the grid and how many tiles its CTAs ran, when each
role's tiles start and end relative to the first CTA, the stage stamps of every role (median / p90 / max since pass start),
how long each stage of a reconcile tile takes and how long its CTA takes from the tile's sweep to its next tile, the shared
decide sub-tiles and the slowest tiles of each role.
python tools/pass_trace.py [C2] [sorted|unsorted]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import kube_throttler_b200 as kt
from kube_throttler_b200 import synth

cfg = sys.argv[1] if len(sys.argv) > 1 else "C2"
sort = not (len(sys.argv) > 2 and sys.argv[2] == "unsorted")
snap = synth.generate(cfg, sort_by_namespace=sort)
eng = kt.Engine(snap.R, snap.L, snap.LN)
eng.upload_snapshot(snap)
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
s = torch.cuda.Stream()
eng.set_stream(s.cuda_stream)
eng.enable_trace(True)
STAGES = {
    "match": [],
    "reconcile": ["rows landed", "2 words evaluated", "barrier", "words+sums", "sweep"],
    "status": ["-", "reconcile seen", "sums read", "status written"],
}
for it in range(4):
    with torch.cuda.stream(s):
        if it >= 2:
            flush.zero_()
            flush.sum()
        eng.evaluate(snap.now)
    torch.cuda.synchronize()
    rows, roles = eng.trace()
    rows = rows.astype(np.float64)
    t0 = rows[:, 2].min()
    grid = int(roles[3])
    cta = rows[:, 28].astype(np.int64)
    per_cta = np.bincount(cta, minlength=grid)
    exit_ = rows[rows[:, 29] > 0, 29]
    span = max(rows[:, 3].max(), exit_.max() if len(exit_) else 0.0)
    print(f"pass {it} ({'cold' if it >= 2 else 'warm'} L2): span {(span - t0) / 1e3:.1f} us, {len(rows)} tiles on {grid} CTAs on {len(set(rows[:, 1]))} SMs; "
          f"tiles per CTA: " + ", ".join(f"{k}: {int((per_cta == k).sum())} CTAs" for k in range(int(per_cta.max()) + 1) if (per_cta == k).any()))
    if len(exit_):
        print(f"  CTA exit  since pass start: med {np.median(exit_ - t0) / 1e3:5.1f}  p90 {np.percentile(exit_ - t0, 90) / 1e3:5.1f}  max {(exit_.max() - t0) / 1e3:5.1f}")
    lo = 0
    for name, n in zip(STAGES, roles[:3]):
        r = rows[lo:lo + int(n)]
        tickets = np.arange(lo, lo + int(n))
        lo += int(n)
        if not len(r):
            continue
        st, en = (r[:, 2] - t0) / 1e3, (r[:, 3] - t0) / 1e3
        print(f"  {name:9s} n={int(n):4d}  start {st.min():5.1f}..{st.max():5.1f}  end med {np.median(en):5.1f} p90 {np.percentile(en, 90):5.1f} max {en.max():5.1f}  dur med {np.median(en - st):5.1f}")
        late = (tickets >= grid) & (name != "status")  # tiles drawn after the first wave: by CTAs that finished an earlier tile
        if late.any():
            print(f"            {int(late.sum())} tiles in the leftover round: start {st[late].min():5.1f}..{st[late].max():5.1f}  end max {en[late].max():5.1f}")
        for k, label in enumerate(STAGES[name]):
            x = (r[:, 4 + k] - t0) / 1e3
            x = x[r[:, 4 + k] > 0]
            if len(x):
                print(f"            {label:18s} since pass start: med {np.median(x):5.1f}  p90 {np.percentile(x, 90):5.1f}  max {x.max():5.1f}")
        if name == "reconcile":  # how long each stage of a tile takes, and what a CTA spends between a tile's sweep and its next tile
            cols = [2] + [4 + k for k in range(len(STAGES[name]))] + [3]
            ok = (r[:, cols] > 0).all(axis=1)
            labels = STAGES[name] + ["end (signal)"]
            parts = [f"{labels[k]} {np.median(d):.2f}/{np.percentile(d, 90):.2f}"
                     for k, d in enumerate((r[ok][:, b] - r[ok][:, a]) / 1e3 for a, b in zip(cols[:-1], cols[1:]))]
            print("            per tile, us since the previous stamp (median/p90): " + " | ".join(parts))
            first = rows[:lo]  # every first-phase tile, in ticket order: a CTA's next tile is its next row
            per_cta_rows = {}
            for i in np.argsort(first[:, 2], kind="stable"):
                per_cta_rows.setdefault(int(first[i, 28]), []).append(i)
            gap_end, gap_sweep = [], []
            for seq in per_cta_rows.values():
                for i, j in zip(seq[:-1], seq[1:]):
                    if lo - int(n) <= i < lo:  # a reconcile tile followed by another first-phase tile on the same CTA
                        gap_end.append(first[j, 2] - first[i, 3])
                        gap_sweep.append(first[j, 2] - first[i, 8])
            if gap_end:
                ge, gs = np.array(gap_end) / 1e3, np.array(gap_sweep) / 1e3
                print(f"            {len(ge)} reconcile tiles followed by another tile on their CTA: end -> next start med {np.median(ge):.2f} "
                      f"p90 {np.percentile(ge, 90):.2f}; sweep -> next start med {np.median(gs):.2f} p90 {np.percentile(gs, 90):.2f} max {gs.max():.2f}")
        if (r[:, 9] > 0).any():  # a CTA's last tile carries the stamps of its first shared decide sub-tile
            sel = r[:, 9] > 0
            print(f"            -> {int(sel.sum())} CTAs whose last tile was one of these went on to shared decide sub-tiles")
            for k, label in enumerate(["rows + pre visible", "slots claimed", "sums seen", "constants done", "decided"]):
                x = (r[sel, 9 + k] - t0) / 1e3
                x = x[r[sel, 9 + k] > 0]
                if len(x):
                    print(f"            decide: {label:18s} since pass start: med {np.median(x):5.1f}  p90 {np.percentile(x, 90):5.1f}  max {x.max():5.1f}")
            # SM cycle counts of thread 0's way through its first sub-tile (check_decide_quad): deltas between consecutive points
            CYC = ["entry", "requests+counters", "word+claim", "ranked+pre asked", "(first dry run)", "sums visible", "pre landed", "constants", "barrier",
                   "pairs decided", "round closed"]
            c = r[sel][:, 16:27].astype(np.int64)
            dry = r[sel][:, 27]
            order = [0, 1, 2, 3, 5, 6, 7, 8, 9, 10]
            parts = []
            for a_, b_ in zip(order[:-1], order[1:]):
                okm = (c[:, a_] > 0) & (c[:, b_] > 0)
                if okm.any():
                    d = c[okm, b_] - c[okm, a_]
                    parts.append(f"{CYC[b_]} {int(np.median(d))}/{int(np.percentile(d, 90))}")
            print("            decide cycles (median/p90 since the previous point): " + " | ".join(parts))
            okm = (c[:, 4] > 0) & (c[:, 3] > 0)
            if okm.any():
                print(f"            dry runs: {int(np.median(dry))} median, {int(dry.max())} max; the first one took {int(np.median(c[okm, 4] - c[okm, 3]))} cycles (median)")
        if it == 3:
            worst = np.argsort(-en)[:4]
            for i in worst:
                stamps = " ".join(f"{(r[i, 4 + k] - t0) / 1e3:5.1f}" if r[i, 4 + k] > 0 else "    -" for k in range(len(STAGES[name])))
                print(f"            slowest: tile {i:4d} sm {int(r[i, 1]):3d} cta {int(r[i, 28]):4d} start {st[i]:5.1f} end {en[i]:5.1f} | {stamps}")
eng.close()
