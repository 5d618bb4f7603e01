"""The integer bound of the int8 fixed-bound pass (q8_dot_bound in coarse_tc.cu), restated in float32 numpy.

The main pass keeps a row of the int8 copy when its int32 accumulator a passes `a > ti`, with ti from one reciprocal per query
(rq = fl(1 / s_q)) and one per tile (rt = fl(1 / s_t)), no division.  The rows it must never drop are those the float test keeps,
fl(fl(s_q s_t) a) > tdot, and through it the key test fl(1 - fl(fl(s_q s_t) a)) < T.  Both are checked here for scales across
the float range, powers of two and the values next to the smallest normal included, and for tdot at and next to integer
multiples of fl(s_q s_t).  The device may contract the loosening `c - |c| 1e-5` into one FMA, so both roundings are checked.
CPU only.
"""
import numpy as np

F = np.float32
INT_MIN = -(2**31)
A_MAX = 2**24  # |accumulator| < 2^24 (127^2 x 1024)


def _bound(tdot, sq, st, fma):
    """q8_dot_bound(tdot, fl(1 / sq), fl(1 / st)), elementwise; returns int64."""
    with np.errstate(all="ignore"):
        rq = F(1) / sq.astype(F)
        rt = F(1) / st.astype(F)
        r = (rq * rt).astype(F)
        f = (tdot.astype(F) * r).astype(F)
        c = np.minimum(np.maximum(f, F(-33554432.0)), F(33554432.0))
        if fma:  # fl(c - |c| * 1e-5f) with one rounding: the float32 product is exact in float64
            x = (c.astype(np.float64) - np.abs(c).astype(np.float64) * np.float64(F(1e-5))).astype(F)
        else:
            x = (c - (np.abs(c) * F(1e-5)).astype(F)).astype(F)
        ti = np.floor(x).astype(np.float64)
        out = np.where(np.isfinite(ti), ti, 0).astype(np.int64) - 1
        bad = np.isnan(f) | ~((r >= F(2.0**-125)) & (r <= F(2.0**125)))
    return np.where(bad, INT_MIN, out)


def _kept_by_float_test(a, sq, st, tdot):
    with np.errstate(all="ignore"):
        sqt = (sq.astype(F) * st.astype(F)).astype(F)
        return (sqt * a.astype(F)).astype(F) > tdot.astype(F)


def _scales():
    s = []
    for e in range(-126, 24, 5):
        for m in (1.0, 1.5, float(np.nextafter(F(2), F(0)))):
            s.append(F(m) * F(2.0**e))
    tiny = F(2.0**-126)
    s += [tiny, np.nextafter(tiny, F(0)), np.nextafter(tiny, F(1)), F(2.0**-149), F(3 * 2.0**-149), F(2.0**-140)]
    s += [F(1.0) / F(127.0), F(1.0) / F(127.0 * np.sqrt(768.0)), F(0.02861), F(3.1e-4)]
    return np.array(s, dtype=F)


def _cases(rng):
    s = _scales()
    sq, st = np.meshgrid(s, s, indexing="ij")
    sq, st = sq.ravel(), st.ravel()
    n = sq.size
    sqt = (sq * st).astype(F)
    out = []
    for a0 in [np.zeros(n), np.ones(n), -np.ones(n), rng.integers(-A_MAX + 1, A_MAX, n), rng.integers(-200, 200, n),
               rng.integers(2**20, 2**23, n)]:
        m = (sqt * a0.astype(F)).astype(F)  # tdot at an integer multiple of fl(s_q s_t), and one ulp either side
        for tdot in (m, np.nextafter(m, F(np.inf)), np.nextafter(m, F(-np.inf))):
            out.append((sq, st, tdot.astype(F)))
    return out


def _check_never_drops(sq, st, tdot, fma):
    ti = _bound(tdot, sq, st, fma)
    # fl(sqt a) is monotone in a, so it is enough that a = ti (or the top of the accumulator range) is not kept
    a = np.clip(ti, -A_MAX, A_MAX)
    kept = _kept_by_float_test(a, sq, st, tdot) & (ti >= -A_MAX)
    assert not kept.any(), list(zip(sq[kept][:5], st[kept][:5], tdot[kept][:5], ti[kept][:5]))
    return ti


def test_bound_never_drops_a_row_the_float_test_keeps():
    rng = np.random.default_rng(5)
    for fma in (False, True):
        for sq, st, tdot in _cases(rng):
            _check_never_drops(sq, st, tdot, fma)


def test_bound_never_drops_a_row_the_key_test_keeps():
    """The chain the kernel relies on: T (a distance) -> tdot = t - (4e-7 + 2.4e-7 |t|), t = 1 - T -> ti; every a with
    fl(1 - fl(sqt a)) < T must pass a > ti.  T at and next to the distances of integer accumulators."""
    rng = np.random.default_rng(6)
    for fma in (False, True):
        for sq, st, _ in _cases(rng)[::3]:
            sqt = (sq * st).astype(F)
            a0 = rng.integers(-A_MAX + 1, A_MAX, sq.size)
            with np.errstate(all="ignore"):
                d0 = (F(1) - (sqt * a0.astype(F)).astype(F)).astype(F)
            for T in (d0, np.nextafter(d0, F(np.inf)), np.nextafter(d0, F(-np.inf))):
                t = (F(1) - T).astype(F)
                slack = (np.float64(F(4e-7)) + np.float64(F(2.4e-7)) * np.abs(t).astype(np.float64)).astype(F) if fma else \
                    (F(4e-7) + (F(2.4e-7) * np.abs(t)).astype(F)).astype(F)
                tdot = (t - slack).astype(F)
                ti = _bound(tdot, sq, st, fma)
                for da in range(-3, 4):
                    a = a0 + da
                    ok = np.abs(a) < A_MAX
                    with np.errstate(all="ignore"):
                        d = (F(1) - (sqt * a.astype(F)).astype(F)).astype(F)
                    kept = ok & (d < T)
                    assert not (kept & ~(a > ti)).any(), (sq[kept & ~(a > ti)][:3], st[kept & ~(a > ti)][:3])


def test_bound_is_tight_for_normal_scales():
    """Conservative is not enough: for the scales of unit rows the bound sits within its loosening of the float test's edge."""
    rng = np.random.default_rng(7)
    n = 20000
    sq = (rng.uniform(1.0 / (127 * 32), 1.0 / 127, n)).astype(F)
    st = (rng.uniform(1.0 / (127 * 32), 1.0 / 127, n)).astype(F)
    tdot = rng.uniform(-1.0, 1.0, n).astype(F)
    for fma in (False, True):
        ti = _check_never_drops(sq, st, tdot, fma)
        sqt = (sq * st).astype(F)
        q = tdot.astype(np.float64) / sqt.astype(np.float64)
        assert (ti > INT_MIN).all()
        assert (np.floor(q) - ti <= 2 + np.abs(q) * 1.1e-5).all()


def test_nan_and_infinite_bounds():
    sq = np.full(3, F(1 / 127.0))
    st = np.full(3, F(1 / 127.0))
    for fma in (False, True):
        ti = _bound(np.array([np.nan, -np.inf, np.inf], dtype=F), sq, st, fma)
        assert ti[0] == INT_MIN  # NaN: everything passes, as before
        assert ti[1] < -A_MAX  # -inf: everything passes
        assert ti[2] >= A_MAX  # +inf (a slot without a query): nothing passes
