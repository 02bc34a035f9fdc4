"""The k-clique oracle (oracle/kclique_oracle.py) against the reference's own CPU
app: against the stored counts (tests/golden/ref_kclique_outputs.json) on every
case of tests/kclique_cases.py, and against the live driver
(oracle/_ref/ref_kclique_driver) when it is built."""
import pytest

from oracle import kclique_oracle as KO
from oracle import refkclique
from tests.kclique_cases import as_indices, kclique_cases, ref_kclique_outputs

REF = ref_kclique_outputs()
CASES = kclique_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference_counts(name):
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    for k, want in REF[name].items():
        if name == "rmat16" and k > 3:   # the set recursion takes minutes there; the GPU test covers it
            continue
        assert KO.count(n, s, d, k) == want, k


def test_reference_counts_cover_the_cases():
    assert set(REF) == set(CASES)
    assert all({3, 4, 5} <= set(v) for v in REF.values())


@pytest.mark.skipif(not refkclique.available(), reason="oracle/_ref/ref_kclique_driver is not built")
@pytest.mark.parametrize("name", ["p2p31", "rmat12", "random5", "shape_multi_loop", "tier_block33"])
def test_live_driver(name):
    n, src, dst, oids = CASES[name]
    for k, want in REF[name].items():
        assert refkclique.run_app(n, src, dst, k, oids=oids) == want, k
