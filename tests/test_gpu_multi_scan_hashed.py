"""The multi-index scan (sptag_b200_multi_scan) with its member iterators on hashed visited sets
(B200.IteratorVisitedSet = 1) that grow during the scan: counts, ids and score bits equal the reference's
(tests/golden/multi_scan) and the per-query stats equal the plain-Python restatement's (tests/oracle_multi_scan.py), as
they do on bitmaps (test_gpu_multi_scan.py)."""
import numpy as np
import pytest

import oracle_multi_scan as oms
import reflib
from sptag_b200 import capi
from test_gpu_multi_scan import close, load_set, params

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _port():
    reflib.build_port()


def opened_table_bytes(g, i, nq, entries):
    """The visited-set bytes of index i's iterator over nq queries at open (sptag_b200_iterator_open_ex): nq tables of
    2^bits entries, bits from `entries` raised until half a table holds the margin, the graph degree + the largest
    duplicate group + 1"""
    graph = np.frombuffer(np.asarray(g["file:%d:graph.bin" % i], np.uint8).tobytes(), np.int32)
    tree = np.frombuffer(np.asarray(g["file:%d:tree.bin" % i], np.uint8).tobytes(), np.int32)
    nodes = tree[2 + tree[0]:2 + tree[0] + 3 * tree[1 + tree[0]]].reshape(-1, 3)
    group = nodes[:, 1] + nodes[:, 2]
    margin = int(graph[1]) + int(group[nodes[:, 1] < -1].max(initial=0)) + 1
    bits = entries.bit_length() - 1
    while (1 << (bits - 1)) < margin:
        bits += 1
    return nq * (4 << bits)


@pytest.mark.parametrize("name", ["dups", "views3"])
def test_multi_scan_on_hashed_iterator_visited_sets(name, tmp_path):
    """Member iterators on hashed visited sets of 64 entries per query, which grow in every scan: the visited-set bytes
    a member holds after the scan differ from what its iterator opened with (a growth adds a buffer, or frees the first
    one once every query moved; these indexes' bitmaps are smaller than the tables)."""
    g, fx, idx = load_set(name, tmp_path)
    try:
        for ix in idx:
            ix.set_param("B200.IteratorVisitedSet", 1)
            ix.set_param("B200.IteratorVisitedHashEntries", 64)
        for p in sorted(key[2:] for key in g.files if key.startswith("k_")):
            k, term, limit, w = params(g, p)
            ids, scores, counts, stats = capi.multi_scan(idx, fx.queries, k, weights=w, term_cond=term, search_limit=limit,
                                                         want_stats=True)
            assert np.array_equal(counts, g["counts_" + p]), p
            assert np.array_equal(ids, g["ids_" + p]), p
            assert np.array_equal(scores.view(np.int32), g["scores_" + p].view(np.int32)), p
            _, _, _, st, _ = oms.expected(fx, k, term, limit, w)
            assert np.array_equal(stats, st), p
            for i, ix in enumerate(idx):
                held = int(ix.get_param("B200.LastIteratorVisitedBytes"))
                assert held != opened_table_bytes(g, i, fx.nq, 64), (p, i)
    finally:
        close(idx)
