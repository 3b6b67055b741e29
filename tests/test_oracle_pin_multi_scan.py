"""CPU pin of the multi-index scan restatement (tests/oracle_multi_scan.py) to the reference's MultiIndexScan outputs
recorded in tests/golden/multi_scan (tests/golden/make_golden_multi_scan.py), and of what those fixtures cover."""
import glob
import os

import numpy as np
import pytest

import oracle_multi_scan as oms
import reflib

HERE = os.path.dirname(os.path.abspath(__file__))
SETS = sorted(glob.glob(os.path.join(HERE, "golden", "multi_scan", "*.npz")))


@pytest.fixture(scope="module", autouse=True)
def _port():
    reflib.build_port()


def cases(g):
    return sorted(key[2:] for key in g.files if key.startswith("k_"))


def weights_of(g, p):
    w = g["weights_" + p]
    return None if w.size == 0 else w


_results = {}


def run_set(path):
    if path not in _results:
        g = np.load(path)
        fx = oms.Fixture(g)
        out = {}
        for p in cases(g):
            out[p] = oms.expected(fx, int(g["k_" + p]), int(g["term_" + p]), int(g["limit_" + p]), weights_of(g, p))
        _results[path] = (g, out)
    return _results[path]


@pytest.mark.parametrize("path", SETS, ids=[os.path.basename(p)[:-4] for p in SETS])
def test_restatement_equals_reference(path):
    g, out = run_set(path)
    for p, (ids, scores, counts, _, _) in out.items():
        assert np.array_equal(counts, g["counts_" + p]), p
        assert np.array_equal(ids, g["ids_" + p]), p
        assert np.array_equal(scores.view(np.int32), g["scores_" + p].view(np.int32)), p


def test_fixtures_cover_the_cases():
    assert len(SETS) == 5
    ends, tie_evictions, output_ties, same_round, naive_differs = set(), 0, 0, 0, 0
    weights, terms0, neg_limits, members, widths = set(), 0, 0, set(), set()
    for path in SETS:
        g, out = run_set(path)
        for p, (_, _, _, stats, res) in out.items():
            ends |= set(stats[:, 3].tolist())
            w = weights_of(g, p)
            weights.add(None if w is None else tuple(w.tolist()))
            terms0 += int(g["term_" + p]) == 0
            neg_limits += int(g["limit_" + p]) < 0
            for r in res:
                tie_evictions += r["tie_evictions"]
                output_ties += len(set(r["scores"].tolist())) < len(r["scores"])
                same_round += r["same_round"]
                naive = [v for _, v in sorted(r["scored"], key=lambda t: t[0])[:len(r["ids"])]]
                naive_differs += naive != r["ids"].tolist()
        fx = oms.Fixture(g)
        members |= {(fx.metric[i], fx.vt[i]) for i in range(fx.n)}
        widths.add(fx.n)
    assert {oms.END_DROPS, oms.END_LIMIT, oms.END_EXHAUSTED} <= ends
    assert terms0 and neg_limits
    assert None in weights and len(weights) >= 4
    assert same_round > 0, "no id was returned by two indexes in one round"
    assert tie_evictions > 0 and output_ties > 0, "equal scores never met at eviction and output"
    assert naive_differs > 0, "a stable sort by score reproduces every output: the heap's tie order is not exercised"
    assert {(0, reflib.VT_FLOAT), (1, reflib.VT_FLOAT), (0, reflib.VT_INT8)} <= members
    # the score's fused tail alone (2, 3), a block of 4 rounded products (5) and a block of 8 (9)
    assert {2, 3, 5, 9} <= widths


def test_sum_equals_unit_weights():
    """rankFunc's sum (weights NULL) and unit weights give the same scores bit for bit"""
    rng = np.random.default_rng(3)
    for n in range(1, 17):
        for _ in range(50):
            d = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(np.float32)
            plain = np.float32(0.0)
            for x in d:
                plain = np.float32(plain + x)
            got = oms.weighted_rank(list(d), [np.float32(1.0)] * n)
            assert np.float32(got).view(np.int32) == plain.view(np.int32)

