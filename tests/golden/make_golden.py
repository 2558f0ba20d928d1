"""Generates tests/golden/*.npz: inputs are re-creatable from (config, kwargs, seed) by the committed generator
(kube_throttler_b200/synth.py), outputs are what the ORACLE (oracle/ko_columnar.h) computes for them.

  python tests/golden/make_golden.py [case ...]     (no case named: all of them)

The reference itself (Go) cannot run in this image (SURVEY.md 8c), so these are oracle outputs, frozen: they pin the
oracle against silent drift (tests/test_golden.py, CPU) and give the CUDA path committed vectors to match bit for bit
(tests/test_golden.py -m gpu) independently of the live oracle build.  The decision vectors transcribed from the reference's
own tests live as literals in tests/test_oracle_kat.py and tests/test_scenarios.py."""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from kube_throttler_b200 import abi, synth  # noqa: E402
from oracle import ko  # noqa: E402

CASES = {
    "c1_example": ("C1", {}, abi.EVAL_FRESH_STATUS),
    "c2_small": ("C2", dict(m=200, n=5000, p=500), abi.EVAL_FRESH_STATUS),
    "c3_mixed_kinds": ("C3", dict(m=300, n=6000, p=800), abi.EVAL_FRESH_STATUS),
    "c3_on_equal": ("C3", dict(m=300, n=6000, p=800), abi.EVAL_ON_EQUAL),
    "c4_overrides": ("C4", dict(m=500, n=8000, p=1000), abi.EVAL_FRESH_STATUS),
    "c2_unsorted_rows": ("C2", dict(m=333, n=7777, p=1111, sort_by_namespace=False), abi.EVAL_FRESH_STATUS),
    "c2_wide_labels_6bit": ("C2", dict(m=200, n=5000, p=700, L=12, q_max=6), abi.EVAL_FRESH_STATUS),
    # requests in [2^44, 2^60 / pods): the third limb of the warp sums, exact-equality thresholds on both sides of the check
    "c2_value_edges": ("C2", dict(m=200, n=5000, p=700, values="wide"), abi.EVAL_FRESH_STATUS),
}
FIELDS = ("admit", "codes", "pend_bitmap", "used", "used_present", "used_cnt", "throttled", "calc_thr", "calc_present", "calc_cnt", "override_active")


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main(names):
    """Writes the named cases (all when none is named); the other entries of index.json stay as they are."""
    path = os.path.join(HERE, "index.json")
    index = json.load(open(path)) if names else {}
    for name, (cfg, kw, flags) in CASES.items():
        if names and name not in names:
            continue
        snap = synth.generate(cfg, **kw)
        res = ko.columnar_evaluate(snap, flags)
        out = {f: getattr(res, f) for f in FIELDS}
        out["run_bitmap_sha256"] = np.frombuffer(bytes.fromhex(digest(res.run_bitmap)), np.uint8)  # the big one: digest only
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        index[name] = dict(config=cfg, kwargs=kw, flags=int(flags), words_per_row=int(res.words_per_row),
                           inputs_sha256=digest(np.concatenate([snap.running.labels.ravel(), snap.running.req.ravel(), snap.pending.labels.ravel(),
                                                                snap.thr.ravel(), snap.req_vals.astype(np.int64)])))
    json.dump(index, open(path, "w"), indent=1, sort_keys=True)
    print("index holds", len(index), "cases")


if __name__ == "__main__":
    main(sys.argv[1:])
