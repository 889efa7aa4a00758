"""-m gpu: the device sampling chain (sampling.cu) stage by stage through its tap (b200_sampler_tap), against the exact twin of
tests/sampler_twin.py over correctly rounded transcendentals -- twin(cr) -- bit for bit: every candidate list, every probability,
typical's entropy, the uniform variate, the drawn position, mirostat 1's k and mirostat's mu.

Where oracle/_ref/libfalcon_chain.so is present, the device's ids are also held to the live reference's.  The reference evaluates
glibc's expf / logf / log2f / powf, which are not correctly rounded, so its ids may differ from the device's where an ulp moves a
value across a boundary; such a difference is explained only when twin(glibc) and twin(cr) draw different ids for that step (the
first stage at which they differ is named).  On these fixed seeds that count is zero.

Case groups (tests/sampling_chain_cases.py) at every row width where the kernel branches (2, 3, 40, 512, 1024 / 1025 for top-k's
rounds against the sort, 4096 / 4097 for the sequential against the chunked draw table, 65,024): distinct rows over several steps
with the window following the drawn ids, and single-step rows with ties, -inf, repeated / out-of-range / +-0 window entries and
probabilities below expf's range.  Typical over zero probabilities has no defined order (the reference's entropy is NaN there): only
a valid id is asked for."""
import numpy as np
import pytest
import sampler_twin as tw
import sampling_chain_cases as sc

pytestmark = pytest.mark.gpu
KEYS = ("top_k", "top_p", "tfs_z", "typical_p", "temp", "repeat_penalty", "frequency_penalty", "presence_penalty", "repeat_last_n",
        "mirostat", "mirostat_tau", "mirostat_eta", "logit_bias")
REF_KEYS = tuple(k for k in KEYS if k != "repeat_last_n")
EXPLAINED = []


def _ref(W, c):
    import refchain
    if not refchain.have_stages() or (W < 40 and c["mirostat"] == 1):       # mirostat 1's N is the context's vocabulary
        return None
    return sc.ref_context(max(W, 40))


def _twins_differ(row, win, c, seed_state, W):
    """the first stage at which twin(glibc) and twin(cr) differ for one step from the same state, or None"""
    mt, mu = seed_state
    a = tw.run(row, win, c, _copy_mt(mt), mu, W, tw.GLIBC)
    b = tw.run(row, win, c, _copy_mt(mt), mu, W, tw.CR)
    d = tw.compare_device(a[2], b[2])
    return (d or "").split(":")[0] if a[0] != b[0] else None


def _copy_mt(mt):
    m = tw.MT19937(0)
    m.mt, m.i = list(mt.mt), mt.i
    return m


def run_case(gpu, W, c, steps_rows, seed):
    """steps_rows: [(row, window)], window None = follow the drawn ids from the first window.  -> list of failures"""
    win = list(steps_rows[0][1])
    dev = gpu.Sampler(gpu.SamplingChain(seed=seed, **{k: c[k] for k in KEYS}), win)
    dev.tap(True)
    ref = _ref(W, c)
    if ref is not None:
        ref.set_seed(seed)
    mt, mu, rmu = tw.MT19937(seed), np.float32(2 * c["mirostat_tau"]), float(np.float32(2 * c["mirostat_tau"]))
    fails = []
    for s, (row, w) in enumerate(steps_rows):
        if w is not None and s > 0:
            raise ValueError("explicit windows are single-step")
        state = (_copy_mt(mt), mu)
        d = gpu.DevBuf(src=np.ascontiguousarray(row, np.float32))
        gid = dev.sample(d.ptr, W)
        got = dev.tap_stages(W)
        tid, mu, want = tw.run(row, win, c, mt, mu, W, tw.CR)
        diff = tw.compare_device(got, want)
        if diff or gid != tid:
            fails.append("step %d: %s (id %d, twin %d)" % (s, diff, gid, tid))
            break
        if ref is not None:
            rid, rmu, _ = ref.sample_chain_stages(row, win, rmu, **{k: c[k] for k in REF_KEYS})
            pen = (want["temp_row"] if "temp_row" in want else want["row"])["logits"]
            if rid != gid and not pen[rid] == pen[gid]:
                stage = _twins_differ(row, win, c, state, W)
                if stage is None:
                    fails.append("step %d: device %d, reference %d, and the twins agree" % (s, gid, rid))
                else:
                    EXPLAINED.append((W, s, gid, rid, stage))
                break                                                  # the windows part from here
        if c["repeat_last_n"] > 0:
            win = (win + [gid])[-c["repeat_last_n"]:]
    dev.free()
    return fails


def _n_random(W):
    return {65024: 3, 4096: 12, 4097: 12}.get(W, 30)


@pytest.mark.parametrize("W", sc.WIDTHS)
def test_device_stages_equal_twin_on_distinct_rows(gpu, W):
    bad = []
    for k, (name, c, steps) in enumerate(sc.distinct_cases(W, _n_random(W))):
        seed = 1000 + k
        win0 = [int(t) for t in np.random.default_rng([W, seed]).integers(0, W, size=c["repeat_last_n"])] if c["repeat_last_n"] else []
        rows = [(sc.wrow(W, seed, s), win0 if s == 0 else None) for s in range(steps)]
        f = run_case(gpu, W, c, rows, seed)
        if f:
            bad.append((name, f[0]))
    assert not bad, bad[:6]


@pytest.mark.parametrize("W", sc.WIDTHS)
def test_device_stages_equal_twin_on_ties_inf_windows_and_spread(gpu, W):
    bad = []
    for k, (name, c, row, win) in enumerate(sc.special_cases(W)):
        f = run_case(gpu, W, c, [(row, win)], 500 + k)
        if f:
            bad.append((name, f[0]))
    assert not bad, bad[:6]


@pytest.mark.parametrize("W", (40, 1024, 65024))
def test_typical_over_zero_probabilities_gives_a_valid_id(gpu, W):
    for name, c, row, win in sc.typical_nan_cases(W):
        dev = gpu.Sampler(gpu.SamplingChain(seed=3, **{k: c[k] for k in KEYS}), win)
        d = gpu.DevBuf(src=row)
        assert all(0 <= dev.sample(d.ptr, W) < W for _ in range(4)), name
        dev.free()


def test_tap_off_leaves_ids_unchanged(gpu):
    """the same seed draws the same ids with the tap on and off; with it off nothing can be read"""
    c = sc._case(top_k=0, tfs_z=0.97, typical_p=0.95, top_p=0.95, temp=1.2)
    rows = [gpu.DevBuf(src=sc.wrow(4097, 5, s)) for s in range(6)]
    ids = []
    for on in (False, True):
        dev = gpu.Sampler(gpu.SamplingChain(seed=21, **{k: c[k] for k in KEYS}))
        dev.tap(on)
        ids.append([dev.sample(r.ptr, 4097) for r in rows])
        if not on:
            with pytest.raises(KeyError):
                dev.tap_stages(4097)
        dev.free()
    assert ids[0] == ids[1]


def test_no_unexplained_or_explained_divergence_from_the_reference():
    """runs after the groups above: every device / reference difference they met, with the stage where the twins part"""
    assert not EXPLAINED, "device ids differ from the reference's where glibc's rounding moves a boundary: %s" % EXPLAINED
