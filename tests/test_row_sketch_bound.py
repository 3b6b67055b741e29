"""The row-sketch bound (tools/row_sketch_model.py sketch_rows / lower_bound, the numpy statement of what
search_kernels.cuh warp_sketch / sketch_lower_bound compute) never exceeds the distance the reference's float distance
function returns, in any of its three summation trees, and says nothing about a vector with a non-finite element."""
import os
import sys

import numpy as np
import pytest

import reflib

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import row_sketch_model as M  # noqa: E402

DIMS = [1, 15, 16, 17, 100, 768, 1000]


def ref_dists(metric, q, rows, width):
    out = np.empty(rows.shape[0], np.float32)
    rows = np.ascontiguousarray(rows, np.float32)
    q = np.ascontiguousarray(q, np.float32)
    L = reflib.ora()
    for i in range(rows.shape[0]):
        out[i] = L.ora_distance(metric, reflib.VT_FLOAT, width, q.ctypes.data, rows[i].ctypes.data, q.shape[0])
    return out


def bounds(metric, q, rows):
    s, sc, er, nr, n2 = M.sketch_rows(rows)
    t, qsc, qer, qnr, qn2 = M.sketch_rows(q[None, :])
    I = s.astype(np.int64) @ t[0].astype(np.int64)
    assert np.abs(I).max(initial=0) <= 127 * 127 * rows.shape[1]
    return M.lower_bound(I.astype(np.int32), (qsc[0], qer[0], qnr[0], qn2[0]), (sc, er, nr, n2), metric == 1, rows.shape[1])


def check(metric, q, rows):
    lb = bounds(metric, q, rows)
    for width in (16, 8, 4):
        d = ref_dists(metric, q, rows, width)
        ok = ~(lb > d)          # a NaN distance is accepted by m_Results: the bound must be -inf there
        ok &= ~(np.isnan(d) & (lb > -np.inf))
        assert ok.all(), (metric, width, rows.shape, lb[~ok][:4], d[~ok][:4])
    return lb


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("dim", DIMS)
def test_random(metric, dim):
    rng = np.random.default_rng(100 * dim + metric)
    for scale in (1.0, 1e-3, 1e4):
        rows = (rng.standard_normal((200, dim)) * scale).astype(np.float32)
        q = (rng.standard_normal(dim) * scale).astype(np.float32)
        if metric == 1:
            rows = reflib.normalize_rows(rows)
            q = reflib.normalize_rows(q[None, :])[0]
        lb = check(metric, q, rows)
        assert np.isfinite(lb).all()
    # the bound is worth having: on 768-d unit vectors it sits within 0.05 of the distance
    if dim == 768 and metric == 1:
        assert (ref_dists(1, q, rows, 16) - lb).max() < 0.05


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("dim", DIMS)
def test_hard_rows(metric, dim):
    rng = np.random.default_rng(7 * dim + metric)
    q = rng.standard_normal(dim).astype(np.float32)
    base = rng.standard_normal((12, dim)).astype(np.float32)
    rows = base.copy()
    rows[0] = 0                                   # zero row
    rows[1] = q                                   # the query itself
    rows[2, 0] = np.float32(1e30)                 # one element far above the rest
    rows[3] *= np.float32(1e-42)                  # denormals
    rows[4] *= np.float32(1e19)                   # products near overflow
    rows[5] = -q
    rows[6, dim // 2] = np.inf
    rows[7, 0] = -np.inf
    rows[8, dim - 1] = np.nan
    rows[9] = np.float32(3e38)
    lb = check(metric, q, rows)
    assert (lb[6:9] == -np.inf).all()             # a non-finite row is never skipped
    zero = np.zeros(dim, np.float32)
    check(metric, zero, rows)
    for bad in (np.inf, np.nan):
        qb = q.copy()
        qb[0] = bad
        assert (check(metric, qb, base) == -np.inf).all()
    big = q.copy()
    big[0] = np.float32(1e30)
    check(metric, big, rows)


@pytest.mark.parametrize("metric", [0, 1])
def test_near_threshold(metric):
    """Rows whose distance is within one ulp to 1e-2 of a threshold: the skip decision `bound > threshold` is never taken
    for a row the reference would keep (distance <= threshold)."""
    rng = np.random.default_rng(5)
    dim = 768
    q = reflib.normalize_rows(rng.standard_normal((1, dim)).astype(np.float32))[0]
    rows = reflib.normalize_rows((q[None, :] + 0.5 * rng.standard_normal((400, dim)) / np.sqrt(dim)).astype(np.float32))
    d = ref_dists(metric, q, rows, 16)
    lb = bounds(metric, q, rows)
    for gap in (0.0, 1e-7, 1e-5, 1e-3, 1e-2):
        for i in range(rows.shape[0]):
            thr = np.float32(d[i] + gap) if gap else d[i]
            assert not lb[i] > thr
            thr_below = np.nextafter(d[i], np.float32(-np.inf))
            assert lb[i] <= d[i] or thr_below < d[i]
    assert (lb <= d).all()


def test_rounding_helpers():
    """The directed fp32 operations of the restatement against exact rational arithmetic."""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    a = (rng.standard_normal(2000) * 10.0 ** rng.integers(-20, 20, 2000)).astype(np.float32)
    b = (rng.standard_normal(2000) * 10.0 ** rng.integers(-20, 20, 2000)).astype(np.float32)
    for up, add, mul in ((True, M.add_ru, M.mul_ru), (False, M.add_rd, M.mul_rd)):
        for got, op in ((add(a, b), lambda x, y: x + y), (mul(a, b), lambda x, y: x * y)):
            for x, y, g in zip(a[:500], b[:500], got[:500]):
                exact = op(Fraction(float(x)), Fraction(float(y)))
                if not np.isfinite(g):
                    continue
                g = np.float32(g)
                if up:
                    assert Fraction(float(g)) >= exact
                    lower = np.nextafter(g, np.float32(-np.inf))
                    assert Fraction(float(lower)) < exact or exact == 0
                else:
                    assert Fraction(float(g)) <= exact
                    upper = np.nextafter(g, np.float32(np.inf))
                    assert Fraction(float(upper)) > exact or exact == 0
