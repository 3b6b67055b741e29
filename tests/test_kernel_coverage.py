"""CPU test: the GPU case matrix of tests/test_gpu_kernel_coverage.py reaches every search-family kernel instantiation the
launch selectors can return.

The reachable set is computed by asking the library's own selectors (sptag_b200_debug_kernel_for: the code the launches
run, no device needed) for every point of their domain: element type, metric, algorithm, dimension class, SimdWidth,
EnableBfs, row sketches, m_Results tier, query slots per SM and kernel family.  A new instantiation or selector branch
without a case fails here, naming the kernel."""
import itertools

import pytest

import reflib
import test_gpu_kernel_coverage as cov

# one representative of each m_Results tier (max(MaxCheck / 16, K)): <= 512, 513-1024, 1025-2048, and beyond
MRES_CAPS = (10, 512, 513, 1024, 1025, 2048, 2049)
DIMS = (128, 768, 27)   # the two specialised dimensions and any other
SLOTS = (0, 14, 16, 17, 20)


def _capi():
    from sptag_b200 import capi
    capi.lib()
    return capi


def reachable():
    """{kernel name: one selector input that reaches it}"""
    capi = _capi()
    out = {}

    def add(**kw):
        name = capi.debug_kernel_for(**kw)
        if name is not None:
            out.setdefault(name, kw)

    for vt, metric, algo, dim, simd, bfs, sketch, mres, slots in itertools.product(
            (reflib.VT_FLOAT, reflib.VT_INT8, reflib.VT_UINT8, reflib.VT_INT16), (0, 1), (capi.ALGO_BKT, capi.ALGO_KDT),
            DIMS, (16, 8), (0, 1), (0, 1), MRES_CAPS, SLOTS):
        add(value_type=vt, metric=metric, algo=algo, dim=dim, simd_width=simd, enable_bfs=bfs, row_sketch=sketch,
            mres_cap=mres, slots=slots, family=capi.FAMILY_SEARCH)
    for bfs, mres in itertools.product((0, 1), MRES_CAPS):  # PQ / OPQ codes: BKT + L2 (PQQuantizer.h:130-136)
        add(value_type=reflib.VT_UINT8, metric=0, algo=capi.ALGO_BKT, dim=8, enable_bfs=bfs, quantized=True,
            mres_cap=mres, family=capi.FAMILY_SEARCH)
    for vt, metric, bfs, mres, fam in itertools.product(
            (reflib.VT_FLOAT, reflib.VT_INT8, reflib.VT_UINT8, reflib.VT_INT16), (0, 1), (0, 1), MRES_CAPS,
            (capi.FAMILY_ITERATE, capi.FAMILY_NEAREST_FIRST)):  # GetIterator is BKT only
        add(value_type=vt, metric=metric, algo=capi.ALGO_BKT, dim=64, enable_bfs=bfs, mres_cap=mres, family=fam)
    return out


def test_every_reachable_instantiation_has_a_case():
    reach = reachable()
    covered = {}
    for c in cov.CASES:
        covered.setdefault(cov.predicted_kernel(c), []).append(cov.case_id(c))
    print("\n%d reachable search-family instantiations:" % len(reach))
    for name in sorted(reach):
        print("  %-70s %s" % (name, ", ".join(covered.get(name, ["-- NO CASE --"]))))
    missing = sorted(set(reach) - set(covered))
    assert not missing, "instantiations no case of tests/test_gpu_kernel_coverage.py runs:\n  " + "\n  ".join(missing)
    assert None not in covered, "cases whose launch no kernel serves: %s" % covered.get(None)
    assert set(covered) <= set(reach)


def test_one_case_per_instantiation():
    """So that removing any case loses an instantiation, which the test above names."""
    seen = {}
    for c in cov.CASES:
        name = cov.predicted_kernel(c)
        assert name not in seen, "%s and %s both run %s" % (seen[name], cov.case_id(c), name)
        seen[name] = cov.case_id(c)


def test_cases_reach_their_tier_with_real_parameters():
    """K and MaxCheck are what the device accepts: K <= 2048 (PQ and iterators 1024), and the k-th result exists."""
    for c in cov.CASES:
        n = {("pq_f32",): 1200, ("pq_opq_i8",): 1500}.get(c.recipe, 1500 if c.recipe[-1] == 768 else cov.N_ROWS)
        assert 1 <= c.k <= n, cov.case_id(c)
        assert max(c.mc // 16, c.k) <= (1024 if c.recipe[0].startswith("pq") or c.family != "search" else 2048)


@pytest.mark.parametrize("family", ["search", "iterate", "nearest"])
def test_selector_refuses_beyond_the_last_tier(family):
    capi = _capi()
    fam = {"search": capi.FAMILY_SEARCH, "iterate": capi.FAMILY_ITERATE, "nearest": capi.FAMILY_NEAREST_FIRST}[family]
    limit = 2048 if family == "search" else 1024
    kw = dict(value_type=reflib.VT_FLOAT, metric=0, algo=capi.ALGO_BKT, dim=64, family=fam)
    assert capi.debug_kernel_for(mres_cap=limit, **kw) is not None
    assert capi.debug_kernel_for(mres_cap=limit + 1, **kw) is None
    assert capi.debug_kernel_for(value_type=reflib.VT_UINT8, metric=0, algo=capi.ALGO_BKT, dim=8, quantized=True,
                                 mres_cap=1025) is None


def compiled_search_kernels():
    """Every compiled search-family instantiation, from the library's exported launch stubs."""
    import re
    import subprocess
    from sptag_b200 import capi
    out = subprocess.run(["nm", "-D", "-C", "--defined-only", capi.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    pat = re.compile(r"\b((?:sptag_b200::)(?:bfs::|sketch::)?(?:search_kernel|iterate_kernel|nearest_first_kernel)<[^>]*>)\(")
    return {m.group(1) for m in pat.finditer(out)}


def test_report_compiled_but_unreachable():
    try:
        compiled = compiled_search_kernels()
    except OSError as e:  # no binutils: nothing to report
        pytest.skip("nm unavailable: %s" % e)
    reach = set(reachable())
    assert reach <= compiled, sorted(reach - compiled)
    print("\ncompiled but unreachable (not tested):")
    for name in sorted(compiled - reach):
        print("  " + name)
