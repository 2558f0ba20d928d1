"""GPU parity: the CUDA path (through the C ABI) against the columnar oracle, bit-exact.

Every output is compared: both match bitmaps, the 2-bit check codes, admit bits, used sums / presence /
counts, throttled masks, calculated thresholds.  Sizes are chosen so the oracle finishes in seconds.
"""
import numpy as np
import pytest

from kube_throttler_b200 import abi, synth

pytestmark = pytest.mark.gpu


def _live(snap):
    return ((snap.thr_flags & abi.THR_RESPONSIBLE) != 0) & ((snap.thr_flags & abi.THR_SELECTOR_ERROR) == 0)


def assert_same(snap, got, want, check_reconcile=True):
    m = snap.m
    assert got.words_per_row == want.words_per_row
    np.testing.assert_array_equal(got.pend_bitmap, want.pend_bitmap, err_msg="pending match bitmap")
    np.testing.assert_array_equal(got.codes, want.codes, err_msg="check codes")
    np.testing.assert_array_equal(got.admit, want.admit, err_msg="admit")
    np.testing.assert_array_equal(got.calc_thr, want.calc_thr, err_msg="calculated threshold")
    np.testing.assert_array_equal(got.calc_present, want.calc_present)
    np.testing.assert_array_equal(got.calc_cnt, want.calc_cnt)
    np.testing.assert_array_equal(got.override_active, want.override_active)
    if check_reconcile:
        live = _live(snap)
        np.testing.assert_array_equal(got.run_bitmap, want.run_bitmap, err_msg="running match bitmap")
        np.testing.assert_array_equal(got.used[:, live], want.used[:, live], err_msg="used")
        np.testing.assert_array_equal(got.used_present[live], want.used_present[live], err_msg="used_present")
        np.testing.assert_array_equal(got.used_cnt[live], want.used_cnt[live], err_msg="used_cnt")
        np.testing.assert_array_equal(got.throttled[live], want.throttled[live], err_msg="throttled")


def run_both(kt, oracle, snap, flags=abi.EVAL_FRESH_STATUS):
    got = kt.evaluate_snapshot(snap, flags)
    want = oracle.columnar_evaluate(snap, flags, words_per_row=got.words_per_row)
    return got, want


def test_c1_example(kt, oracle):
    snap = synth.generate("C1")
    got, want = run_both(kt, oracle, snap)
    assert_same(snap, got, want)
    assert list(got.code_matrix(1)[:, 0]) == [0, 2, 3]  # 100m admit, 101m insufficient, 300m exceeds
    assert list(got.admit) == [1, 0, 0]
    assert got.used[0, 0] == 100 and got.used_cnt[0] == 10


@pytest.mark.parametrize("kw", [
    dict(config="C2", m=64, n=3000, p=400),
    dict(config="C2", m=200, n=5000, p=500),
    dict(config="C2", m=1000, n=20000, p=2000),
    dict(config="C2", m=333, n=7777, p=1111, sort_by_namespace=False),
    dict(config="C3", m=300, n=6000, p=800),
    dict(config="C3", m=1000, n=20000, p=2000),
    dict(config="C4", m=500, n=8000, p=1000),
    dict(config="C3", m=1000, n=20000, p=2000, sort_by_namespace=False),  # > kSlots distinct words per CTA: direct REDs
    dict(config="C2", m=150, n=4000, p=600, R=12),                        # R > 8: shared-memory accumulation variant
    dict(config="C2", m=40, n=70, p=33, R=1),                             # ragged: partial tiles, partial last word
    dict(config="C3", m=200, n=5000, p=700, L=12),                        # L > 8: label rows staged in shared memory
    dict(config="C2", m=200, n=5000, p=700, L=12, q_max=6),               # terms with > 3 required keys: 6-bit counters
    dict(config="C3", m=120, n=2000, p=300, R=31, L=16),                  # the limits: every resource bit in use, two label chunks
    dict(config="C3", m=64, n=3000, p=400, L=3, R=2),                     # fewer label slots than a chunk
    dict(config="C3", m=300, n=6000, p=800, column_layout=True),          # ClusterThrottles in the host layer's column order (by namespace set)
    dict(config="C2", m=150, n=300, p=6000),                              # far more pending than running rows: 50 CTAs serve ~200 decide sub-tiles / status tiles
    dict(config="C3", m=400, n=500, p=5000, sort_by_namespace=False),     # the same with ClusterThrottles and rows in arrival order: several rounds per sub-tile, pairs checked straight from L2
] + [  # request values at the edges of the 64-bit sums (synth.VALUE_REGIMES) through the register (R=4), direct-RED (R=8, more
    # distinct words than slots) and shared-memory (R=12) accumulation paths
    dict(kw, values=v) for v in synth.VALUE_REGIMES for kw in (
        dict(config="C2", m=200, n=5000, p=700),
        dict(config="C3", m=1000, n=20000, p=2000, sort_by_namespace=False),
        dict(config="C2", m=150, n=4000, p=600, R=12))
])
def test_scaled_configs(kt, oracle, kw):
    kw = dict(kw)
    snap = synth.generate(kw.pop("config"), **kw)
    got, want = run_both(kt, oracle, snap)
    assert_same(snap, got, want)
    assert got.match_matrix("pending", snap.m).sum() > 0


def _remap_label_ids(snap, kf, vf):
    """Re-number label key / value dictionary ids everywhere they occur (pods, namespaces, selectors)."""
    def remap(lab):
        key, val = lab >> 32, lab & 0xFFFFFFFF
        return np.where(lab == abi.LABEL_EMPTY, abi.LABEL_EMPTY, (kf(key) << 32) | vf(val)).astype(np.int64)
    for pods in (snap.running, snap.pending):
        pods.labels = np.ascontiguousarray(remap(pods.labels))
    snap.ns_labels = np.ascontiguousarray(remap(snap.ns_labels))
    snap.req_key = kf(snap.req_key.astype(np.int64)).astype(np.uint32)
    snap.req_vals = vf(snap.req_vals.astype(np.int64)).astype(np.uint32)
    return snap.normalize()


@pytest.mark.parametrize("mode", ["sparse_keys", "sparse_values"])
def test_sparse_dictionary_ids(kt, oracle, mode):
    """Label ids are opaque: ids too sparse for the direct key/value tables take the hashed lookup."""
    snap = synth.generate("C3", m=300, n=6000, p=800)
    base = kt.evaluate_snapshot(snap)
    if mode == "sparse_keys":  # key ids beyond the direct key table: every label is hashed
        snap = _remap_label_ids(snap, lambda k: k * 7919 + 70000, lambda v: v * 1009 + 5)
    else:                      # small key ids, value ids spread out: per-key hashed values
        snap = _remap_label_ids(snap, lambda k: k, lambda v: v * 1000003 % (1 << 31))
    got, want = run_both(kt, oracle, snap)
    assert_same(snap, got, want)
    # a pure renaming of ids must not change any decision
    np.testing.assert_array_equal(got.codes, base.codes)
    np.testing.assert_array_equal(got.used, base.used)


@pytest.mark.parametrize("values", (None,) + synth.VALUE_REGIMES)
def test_on_equal_flag(kt, oracle, values):
    snap = synth.generate("C3", m=300, n=6000, p=800, values=values)
    got, want = run_both(kt, oracle, snap, abi.EVAL_ON_EQUAL)
    assert_same(snap, got, want)


@pytest.mark.parametrize("values", (None,) + synth.VALUE_REGIMES)
def test_given_status(kt, oracle, values):
    """PreFilter between reconciles: the check uses an uploaded (stale) status, not this pass's."""
    snap = synth.generate("C4", m=400, n=6000, p=900, values=values)
    fresh = oracle.columnar_evaluate(snap)
    rng = np.random.default_rng(7)
    m, R = snap.m, snap.R
    st = dict(calculated=(rng.random(m) < 0.8).astype(np.uint8), calc_thr=fresh.calc_thr.copy(), calc_present=fresh.calc_present.copy(),
              calc_cnt=fresh.calc_cnt.copy(), used=fresh.used.copy(), used_present=fresh.used_present.copy(),
              used_cnt=fresh.used_cnt.copy(), throttled=fresh.throttled.copy())
    # make it stale: perturb used on a third of the throttles, drop throttled bits on some
    stale = rng.random(m) < 0.33
    st["used"][:, stale] = (st["used"][:, stale] * 0.5).astype(np.int64)
    st["throttled"][rng.random(m) < 0.2] = 0
    snap.status = st
    snap.normalize()
    for flags in (abi.EVAL_GIVEN_STATUS, abi.EVAL_GIVEN_STATUS | abi.EVAL_ON_EQUAL, abi.EVAL_GIVEN_STATUS | abi.EVAL_SKIP_RECONCILE):
        got, want = run_both(kt, oracle, snap, flags)
        assert_same(snap, got, want, check_reconcile=not (flags & abi.EVAL_SKIP_RECONCILE))


def test_c2_full_size(kt, oracle):
    """BASELINE config 2 at full size (1k x 100k x 10k): the oracle needs ~1 s for it."""
    snap = synth.generate("C2")
    got, want = run_both(kt, oracle, snap)
    assert_same(snap, got, want)
    used, present, cnt = snap.meta["true_used"]  # third implementation (numpy)
    live = _live(snap)
    np.testing.assert_array_equal(got.used[:, live], used[:, live])
    np.testing.assert_array_equal(got.used_cnt[live], cnt[live])


@pytest.mark.parametrize("config,kw", [
    ("C2", dict(sort_by_namespace=False)),   # arrival-order rows: the multi-word / direct-RED path at full size
    ("C3", dict()),                          # 600 Throttles + 400 ClusterThrottles with namespace selectors, R=8
    ("C3", dict(sort_by_namespace=False)),
    ("C4", dict()),                          # 5k throttles, temporaryThresholdOverrides active on 20 %
    ("C5", dict()),                          # 10k x 1M x 100k on ONE GPU (1.9 GB); the columnar oracle needs ~1 min
])
def test_baseline_configs_full_size(kt, oracle, config, kw):
    """Every BASELINE.json config at its FULL size on one device, every output bit against the columnar oracle
    (C1 and sorted C2 are test_c1_example / test_c2_full_size)."""
    snap = synth.generate(config, **kw)
    got, want = run_both(kt, oracle, snap)
    assert_same(snap, got, want)
    assert got.pend_bitmap.any() and got.run_bitmap.any()


def test_repeat_pass_is_idempotent(kt):
    """The partial-sum buffer is consumed and re-zeroed by every pass: two passes give identical results."""
    snap = synth.generate("C2", m=200, n=5000, p=500)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    eng.evaluate(snap.now)
    a = eng.download()
    eng.evaluate(snap.now)
    b = eng.download()
    for f in ("used", "used_cnt", "used_present", "throttled", "codes", "admit", "run_bitmap", "pend_bitmap"):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f)
    eng.close()


@pytest.mark.parametrize("values", (None,) + synth.VALUE_REGIMES)
def test_fused_and_chained_paths_agree(kt, oracle, values):
    """kt_evaluate runs the whole pass as ONE launch (k_pass: ticketed reconcile / finalize / check tiles with in-kernel
    hand-offs); with per-kernel timing enabled it runs the three PDL-chained kernels instead.  Same bits either way,
    pass after pass (the ticket / done counters re-arm themselves)."""
    for kw in (dict(config="C3", m=300, n=6000, p=800), dict(config="C2", m=1000, n=30000, p=3000), dict(config="C2", m=40, n=70, p=33, R=1)):
        kw = dict(kw, values=values)
        snap = synth.generate(kw.pop("config"), **kw)
        eng = kt.Engine(snap.R, snap.L, snap.LN)
        eng.upload_snapshot(snap)
        outs = []
        for timing in (False, False, True, False):
            eng.enable_timing(timing)
            eng.evaluate(snap.now)
            outs.append(eng.download())
            assert eng.timing().launches == (3 if timing else 1)
        eng.close()
        want = oracle.columnar_evaluate(snap, words_per_row=outs[0].words_per_row)
        for got in outs:
            assert_same(snap, got, want)


def test_compact_upload_equals_wide_upload(kt, oracle):
    """kt_upload_pods_compact expands to exactly the int64 columns kt_upload_pods would have copied: same bits out."""
    for kw in (dict(config="C3", m=300, n=6000, p=800), dict(config="C2", m=200, n=5000, p=700, L=12), dict(config="C2", m=40, n=70, p=33, R=1, L=3)):
        kw = dict(kw)
        snap = synth.generate(kw.pop("config"), **kw)
        eng = kt.Engine(snap.R, snap.L, snap.LN)
        eng.upload_snapshot(snap)
        for kind, pods in ((abi.PODS_RUNNING, snap.running), (abi.PODS_PENDING, snap.pending)):
            cp = abi.compact_pods(pods)
            assert cp.nbytes < 0.6 * sum(a.nbytes for a in (pods.labels, pods.req, pods.present, pods.flags, pods.ns_id))
            eng.upload_pods_compact(kind, cp)
        eng.evaluate(snap.now)
        got = eng.download()
        eng.close()
        want = oracle.columnar_evaluate(snap, words_per_row=got.words_per_row)
        assert_same(snap, got, want)
    bad = synth.generate("C2", m=40, n=70, p=33).running
    bad.req[0, 3] = (1 << 40) + 1  # odd and huge: no power-of-two unit makes the column fit int32
    with pytest.raises(ValueError):
        abi.compact_pods(bad)
    bad = synth.generate("C2", m=40, n=70, p=33).running
    bad.labels[0, 0] = (5 << 32) | (1 << 25)  # value id beyond the 20-bit split
    with pytest.raises(ValueError):
        abi.compact_pods(bad)


def test_pod_row_delta(kt, oracle):
    """kt_update_pod_rows == re-uploading the modified columns (informer Add/Update/Delete as row scatters)."""
    snap = synth.generate("C2", m=200, n=5000, p=500)
    other = synth.generate("C2", m=200, n=5000, p=500, seed=99)
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    rng = np.random.default_rng(3)
    rows = np.sort(rng.choice(snap.running.n, size=600, replace=False)).astype(np.int64)
    delta = other.running.rows(rows)
    delta.flags[:50] = 0  # deleted pods: never counted
    delta.labels[:, :50] = abi.LABEL_EMPTY
    eng.update_pod_rows(abi.PODS_RUNNING, rows, delta)
    eng.evaluate(snap.now)
    got = eng.download()
    eng.close()
    for name in ("labels", "req"):
        getattr(snap.running, name)[:, rows] = getattr(delta, name)
    for name in ("present", "flags", "ns_id"):
        getattr(snap.running, name)[rows] = getattr(delta, name)
    want = oracle.columnar_evaluate(snap, words_per_row=got.words_per_row)
    assert_same(snap, got, want)


def test_no_gpu_error_contract(kt):
    """Calls out of order fail with KT_ERR_STATE, never with a silent default."""
    eng = kt.Engine(4, 8, 4)
    with pytest.raises(kt.KtError) as e:
        eng.evaluate(0)
    assert e.value.code == abi.ERR_STATE
    eng.close()


@pytest.mark.parametrize("values", (None,) + synth.VALUE_REGIMES)
def test_packed_upload_equals_wide_upload(kt, oracle, values):
    """kt_upload_pods_packed (16-bit label-pair indices, presence in the meta word) expands to exactly the int64 columns
    kt_upload_pods would have copied: same bits out.  Requests beyond int32 (the value regimes) travel dictionary-coded; the
    int32 packer refuses them."""
    for kw in (dict(config="C3", m=300, n=6000, p=800), dict(config="C2", m=200, n=5000, p=700, L=12), dict(config="C2", m=40, n=70, p=33, R=1, L=3),
               dict(config="C4", m=500, n=3000, p=400)):
        kw = dict(kw, values=values)
        snap = synth.generate(kw.pop("config"), **kw)
        eng = kt.Engine(snap.R, snap.L, snap.LN)
        eng.upload_snapshot(snap)
        want = None
        for coded in (False, True):  # int32 request columns, then dictionary-coded ones
            if values is not None and not coded:
                for pods in (snap.running, snap.pending):
                    with pytest.raises(ValueError):
                        abi.packed_pods(pods, code_requests=False)
                continue
            for kind, pods in ((abi.PODS_RUNNING, snap.running), (abi.PODS_PENDING, snap.pending)):
                pk = abi.packed_pods(pods, code_requests=coded)
                if pods.n >= 1000 and values is None:  # the pair dictionary is a fixed cost: only rows amortise it
                    assert pk.nbytes < 0.65 * sum(a.nbytes for a in (pods.labels, pods.req, pods.present, pods.flags, pods.ns_id))
                eng.upload_pods_packed(kind, pk)
            eng.evaluate(snap.now)
            got = eng.download()
            want = want or oracle.columnar_evaluate(snap, words_per_row=got.words_per_row)
            assert_same(snap, got, want)
        eng.close()


@pytest.mark.parametrize("fused", [True, False])
def test_sparse_check_equals_nonzero_words_of_the_dense_rows(kt, oracle, fused):
    """kt_get_check_sparse: exactly the non-zero code words of kt_get_check, each once, plus the same admit bits; a list
    that is too small reports the true count so that the caller can fall back to the dense rows."""
    for kw in (dict(config="C2", m=300, n=8000, p=1500), dict(config="C3", m=200, n=3000, p=700), dict(config="C2", m=40, n=70, p=33, R=1, L=3)):
        kw = dict(kw)
        snap = synth.generate(kw.pop("config"), **kw)
        eng = kt.Engine(snap.R, snap.L, snap.LN)
        eng.upload_snapshot(snap)
        eng.set_sparse_check(4 * snap.pending.n + 64)
        if not fused:
            eng.enable_timing(True)  # per-kernel events: the three chained kernels instead of the one fused launch
        for _ in range(2):  # twice: the counter is cleared by the pass itself
            eng.evaluate(snap.now)
            got = eng.download()
            Wp = got.words_per_row
            ent = np.zeros((4 * snap.pending.n + 64, 3), np.uint32)
            admit = np.zeros(snap.pending.n, np.uint8)
            cnt = eng.get_check_sparse(admit, ent)
            dense = got.codes.reshape(snap.pending.n, 2 * Wp)
            rows, widx = np.nonzero(dense)
            assert cnt == rows.shape[0]
            want = sorted(zip(rows.tolist(), widx.tolist(), dense[rows, widx].tolist()))
            assert sorted(map(tuple, ent[:cnt].tolist())) == want
            assert np.array_equal(admit, got.admit)
        small = np.zeros((max(cnt // 2, 1), 3), np.uint32)
        assert eng.get_check_sparse(None, small) == cnt  # truncated: the count still says how many there are
        eng.set_sparse_check(0)
        eng.evaluate(snap.now)
        with pytest.raises(Exception):
            eng.get_check_sparse(None, small)
        eng.close()


def test_device_side_status_diff(kt, oracle):
    """SURVEY 8f.3: with an observed status uploaded, the reconciling pass itself says which throttles' status it changes
    (throttle_controller.go:157 DeepEqual) -- compared here with a numpy diff of the oracle's outputs against the same observed
    status -- and kt_get_reconcile_rows / kt_get_check_rows deliver exactly the listed rows of the full downloads."""
    snap = synth.generate("C4", m=700, n=9000, p=1200)
    fresh = oracle.columnar_evaluate(snap)
    rng = np.random.default_rng(11)
    m, R = snap.m, snap.R
    st = dict(calculated=(rng.random(m) < 0.9).astype(np.uint8), calc_thr=fresh.calc_thr.copy(), calc_present=fresh.calc_present.copy(),
              calc_cnt=fresh.calc_cnt.copy(), used=fresh.used.copy(), used_present=fresh.used_present.copy(),
              used_cnt=fresh.used_cnt.copy(), throttled=fresh.throttled.copy())
    # the informer copy lags: other sums on a fifth of the throttles, a flipped throttled bit, a stale threshold, a lost key
    a, b, c_, d = (rng.random(m) < 0.2), (rng.random(m) < 0.05), (rng.random(m) < 0.05), (rng.random(m) < 0.05)
    st["used"][0, a] += 7
    st["throttled"][b] ^= 1
    st["calc_thr"][min(1, R - 1), c_] += 1
    st["used_present"][d] &= ~np.uint32(1)
    snap.status = st
    snap.normalize()
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    for _ in range(2):  # twice: the list counter re-arms itself
        eng.evaluate(snap.now)
        got = eng.download()
        idx, flags = eng.get_changed()
        live = _live(snap)
        pm = lambda x: x[None, :] if x.ndim == 1 else x
        differs = np.zeros(m, bool)
        R_bits = (np.uint32(1) << np.arange(R, dtype=np.uint32))[:, None]
        for name_v, name_p, cnt in (("used", "used_present", "used_cnt"), ("calc_thr", "calc_present", "calc_cnt")):
            gp, sp = getattr(got, name_p), st[name_p]
            differs |= gp != sp
            has = (gp[None, :] & R_bits) != 0
            differs |= ((getattr(got, name_v) != st[name_v]) & has).any(axis=0)
            differs |= (getattr(got, cnt) != st[cnt]) & ((gp & abi.COUNT_BIT) != 0)
        differs |= got.throttled != st["throttled"]
        differs |= st["calculated"] == 0
        differs &= live
        np.testing.assert_array_equal(flags.astype(bool), differs)
        np.testing.assert_array_equal(idx, np.nonzero(differs)[0])
        assert 0 < idx.shape[0] < m
        rows = eng.get_reconcile_rows(idx)
        for f in ("used", "calc_thr"):
            np.testing.assert_array_equal(getattr(rows, f), getattr(got, f)[:, idx], err_msg=f)
        for f in ("used_present", "used_cnt", "throttled", "calc_present", "calc_cnt", "override_active"):
            np.testing.assert_array_equal(getattr(rows, f), getattr(got, f)[idx], err_msg=f)
        pick = np.sort(rng.choice(snap.pending.n, size=77, replace=False)).astype(np.int64)
        codes, admit = eng.get_check_rows(pick)
        np.testing.assert_array_equal(codes, got.codes[pick])
        np.testing.assert_array_equal(admit, got.admit[pick])
    eng.close()


def test_step_api_equals_separate_calls(kt, oracle):
    """kt_step_submit / kt_step_wait: one call queues packed uploads + pass + result copies, one synchronisation delivers the
    status columns, admit bits and non-zero code words in one pinned block -- the same bits as the separate calls, step
    after step, also with two contexts alternating (double buffering) and with the resident rows kept (NULL uploads)."""
    import ctypes as C

    def view(ptr, dtype, shape):
        n = int(np.prod(shape))
        if n == 0:
            return np.zeros(shape, dtype)
        buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape).copy()

    snaps = [synth.generate("C2", m=300, n=8000, p=1500), synth.generate("C2", m=300, n=8000, p=1500, seed=77)]
    want = []
    engines = []
    for snap in snaps:
        eng = kt.Engine(snap.R, snap.L, snap.LN)
        eng.upload_snapshot(snap)
        eng.set_sparse_check(4 * snap.pending.n + 64)
        engines.append(eng)
        got = None
    packed = [[abi.packed_pods(pods, code_requests=True) for pods in (s_.running, s_.pending)] for s_ in snaps]
    # the second snapshot's columns are carved out of ONE host block per kind: the library detects it and sends one transfer
    blocks = []
    for k, c in enumerate(packed[1]):
        arrays = [c.labels16, c.pairs, c.meta, c.req_codes, c.req_dict]
        offs, at = [], 0
        for a in arrays:
            offs.append(at)
            at += (a.nbytes + 15) & ~15
        blk = kt.Pinned((at,), np.uint8)
        blocks.append(blk)
        views = []
        for a, o in zip(arrays, offs):
            v = blk.array[o:o + a.nbytes].view(a.dtype).reshape(a.shape)
            v[...] = a
            views.append(v)
        packed[1][k] = abi.PackedPodCols(c.ns_bits, views[1], views[0], None, None, views[2], views[4], c.req_dict_off, c.req_code_bytes, views[3])
    for it in range(4):
        for eng, snap, pk in zip(engines, snaps, packed):  # both submitted before either is waited for
            if it == 3:
                eng.step_submit(None, None, snap.now)  # resident rows
            else:
                eng.step_submit(pk[0], pk[1], snap.now)
        for eng, snap in zip(engines, snaps):
            res = eng.step_wait()
            W = eng.words_per_row
            ref = oracle.columnar_evaluate(snap, words_per_row=W)
            P, m, R = snap.pending.n, snap.m, snap.R
            assert res.n_pending == P
            np.testing.assert_array_equal(view(res.admit, np.uint8, (P,)), ref.admit)
            ent = view(res.entries, np.uint32, (int(res.n_sparse), 3))
            dense = np.zeros((P, 2 * W), np.uint32)
            dense[ent[:, 0], ent[:, 1]] = ent[:, 2]
            np.testing.assert_array_equal(dense, ref.codes)
            assert len({(a, b) for a, b in ent[:, :2].tolist()}) == ent.shape[0]
            live = _live(snap)
            st = res.status
            np.testing.assert_array_equal(view(st.used, np.int64, (R, m))[:, live], ref.used[:, live])
            np.testing.assert_array_equal(view(st.used_cnt, np.int64, (m,))[live], ref.used_cnt[live])
            np.testing.assert_array_equal(view(st.used_present, np.uint32, (m,))[live], ref.used_present[live])
            np.testing.assert_array_equal(view(st.throttled, np.uint32, (m,))[live], ref.throttled[live])
            np.testing.assert_array_equal(view(st.calc_thr, np.int64, (R, m)), ref.calc_thr)
            np.testing.assert_array_equal(view(st.calc_present, np.uint32, (m,)), ref.calc_present)
    for eng in engines:
        eng.close()


C2Q = dict(config="C2", m=200, n=4000, p=2600)


@pytest.mark.parametrize("world,first,count,flags", [
    (dict(config="C2", m=200, n=4000, p=1000), 0, None, 0),
    (dict(config="C3", m=120, n=3000, p=600, seed=9), 0, None, 0),
    (C2Q, 0, 1, 0),                  # queue lengths around one CSR block (kAdmitBlock = 1024 queue positions)
    (C2Q, 0, 1023, 0),
    (C2Q, 0, 1024, 0),
    (C2Q, 0, 1025, 0),
    (C2Q, 0, 2500, 0),
    (C2Q, 41, 1025, 0),              # a sub-range of the pending table: the rows around it keep the pass's codes and admit bits
    (C2Q, 1500, 1024, abi.EVAL_ON_EQUAL),
    (dict(config="C4", m=2500, n=20000, p=1500), 0, None, 0),  # M > 1024: k_admit_starts scans ranges; overrides active
    (dict(config="C2", m=200, n=4000, p=1000, R=1), 0, None, 0),            # each k_admit_round<RMAX>, and the first R past each bound
    (dict(config="C3", m=200, n=3000, p=800, R=5), 0, None, 0),
    (dict(config="C3", m=200, n=3000, p=800, R=9), 0, None, abi.EVAL_ON_EQUAL),
    (dict(config="C3", m=120, n=2000, p=600, R=31, L=16), 0, None, 0),
    (dict(config="C3", m=120, n=3000, p=600, seed=9), 0, None, abi.EVAL_ON_EQUAL),
    (dict(config="C2", m=200, n=4000, p=1000, throttled=True, zero_counts=True), 0, None, 0),
    (dict(config="C2", m=200, n=4000, p=1000, orphans=True), 0, None, 0),   # pods that affect no throttle
    (dict(config="C2", m=200, n=4000, p=1500, values="signed"), 0, None, 0),
    (dict(config="C3", m=200, n=3000, p=1200, values="signed"), 100, 1000, abi.EVAL_ON_EQUAL),
])
def test_device_queue_admission_equals_pod_by_pod(kt, oracle, world, first, count, flags):
    """SURVEY 8f.2: kt_admit_queue (per-throttle prefix sums over the admitted pods, iterated to the fixpoint on the device) gives
    every pod of the queue the verdict and the check codes it gets when the queue is admitted ONE POD PER CYCLE -- PreFilter
    against observed status + reservations, Reserve on Success (plugin.go:148-238) -- as the columnar oracle's
    columnar_admit_queue walks it; the pending rows outside the queue keep the codes of a GIVEN_STATUS | SKIP_RECONCILE pass."""
    from test_oracle_admission import FLAGS, admission_world

    world = dict(world)
    snap = admission_world(oracle, world.pop("config"), **world)
    P = snap.pending.n
    count = P - first if count is None else count
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    rounds, admitted = eng.admit_queue(first, count, flags)
    got = eng.download()
    eng.close()
    want, n_adm, _ = oracle.columnar_admit_queue(snap, first, count, flags, words_per_row=got.words_per_row)
    np.testing.assert_array_equal(got.pend_bitmap, want.pend_bitmap)
    np.testing.assert_array_equal(got.admit, want.admit)
    np.testing.assert_array_equal(got.codes, want.codes)
    assert admitted == n_adm
    if first > 0 or first + count < P:  # the rows outside the queue, once more against the plain pass
        out = np.ones(P, bool)
        out[first:first + count] = False
        plain = oracle.columnar_evaluate(snap, FLAGS | flags, words_per_row=got.words_per_row)
        np.testing.assert_array_equal(got.codes[out], plain.codes[out])
        np.testing.assert_array_equal(got.admit[out], plain.admit[out])
    if count >= 500:
        assert 0.05 * count < n_adm < 0.95 * count, (n_adm, count)  # not degenerate
    assert 2 <= rounds <= 64, rounds


def _two_pod_world():
    """T1: cpu threshold 10, observed used 5.  T2: pod: 0.  Queue: A (cpu -5, on T1 and T2), then B (cpu 8, on T1)."""
    L, R, LN = 2, 1, 1
    lab = np.full((L, 2), abi.LABEL_EMPTY, np.int64)
    lab[0] = (np.int64(0) << 32) | 0                 # k0=v0: both pods (T1's selector)
    lab[1, 0] = (np.int64(1) << 32) | 0              # k1=v0: A only (T2's selector)
    pending = abi.PodCols(lab, np.array([[-5, 8]], np.int64), np.ones(2, np.uint32), np.full(2, abi.POD_SCHEDULER_MATCH | abi.POD_NOT_FINISHED, np.uint32),
                          np.zeros(2, np.int32))
    running = abi.PodCols(np.full((L, 0), abi.LABEL_EMPTY, np.int64), np.zeros((R, 0), np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32),
                          np.zeros(0, np.int32))
    sel = synth.build_selector_csr([0, 1, 2], [[(0, abi.OP_IN, [0])], [(1, abi.OP_IN, [0])]], [[], []])
    thr, thr_present, thr_cnt = np.array([[10, 0]], np.int64), np.array([1, abi.COUNT_BIT], np.uint32), np.array([0, 0], np.int64)
    snap = abi.Snapshot(
        R=R, L=L, LN=LN, running=running, pending=pending, ns_labels=np.full((LN, 1), abi.LABEL_EMPTY, np.int64),
        kind=np.zeros(2, np.uint8), thr_ns=np.zeros(2, np.int32), thr_flags=np.full(2, abi.THR_RESPONSIBLE, np.uint8),
        thr=thr, thr_present=thr_present, thr_cnt=thr_cnt,
        ovr_off=np.zeros(3, np.int32), ovr_begin=np.zeros(0, np.int64), ovr_end=np.zeros(0, np.int64),
        ovr_flags=np.zeros(0, np.uint8), ovr_thr=np.zeros((R, 0), np.int64), ovr_present=np.zeros(0, np.uint32),
        ovr_cnt=np.zeros(0, np.int64), now=synth.NOW_2026, **sel)
    snap.status = dict(calculated=np.ones(2, np.uint8), calc_thr=thr.copy(), calc_present=thr_present.copy(), calc_cnt=thr_cnt.copy(),
                       used=np.array([[5, 0]], np.int64), used_present=np.array([1 | abi.COUNT_BIT, 0], np.uint32),
                       used_cnt=np.array([1, 0], np.int64), throttled=np.zeros(2, np.uint32))
    return snap.normalize()


def test_device_queue_admission_with_a_negative_request(kt, oracle):
    """A negative undecided request lowers the load the pods behind it see.  One pod per cycle: A is rejected (S1 on T2's pod
    count of 0), so B sees 5 + 8 > 10 on T1 and is insufficient.  Bounding the load from above by "Admitted + Undecided" let B
    see 5 - 5 + 8 and admitted it."""
    snap = _two_pod_world()
    want, n_adm, _ = oracle.columnar_admit_queue(snap, 0, 2, 0, words_per_row=4)
    assert list(want.admit) == [0, 0] and n_adm == 0
    assert list(want.code_matrix(2)[:, 0]) == [0, abi.CHECK_INSUFFICIENT] and want.code_matrix(2)[0, 1] == abi.CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD
    eng = kt.Engine(snap.R, snap.L, snap.LN)
    eng.upload_snapshot(snap)
    rounds, admitted = eng.admit_queue(0, 2)
    got = eng.download()
    eng.close()
    np.testing.assert_array_equal(got.admit, want.admit)
    np.testing.assert_array_equal(got.codes, want.codes)
    assert admitted == 0
