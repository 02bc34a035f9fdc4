"""The directed LCC oracle's reference mode (oracle/lcc_directed_oracle.py, reference=True: uint8_t
weights) against the reference's own LCCDirected: bit for bit against the stored digests of its tri and
deduplicated-degree arrays (tests/golden/ref_lcc_directed_outputs.json) on every case of
tests/lcc_directed_cases.py, and against the live driver (oracle/_ref/ref_lcc_directed_driver) when it
is built."""
import numpy as np
import pytest

from oracle import lcc_directed_oracle as LO
from oracle import reflccd
from tests import golden_io as G
from tests.lcc_directed_cases import WRAP, as_indices, lcc_directed_cases, ref_lcc_directed_outputs

REF = ref_lcc_directed_outputs()
CASES = lcc_directed_cases()


def oracle(name, reference):
    n, src, dst, oids = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    return LO.lcc_directed(n, s, d, reference=reference)


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_mode_equals_digests(name):
    _, tri, d = oracle(name, True)
    assert G.digest(tri) == REF[name]["tri"]
    assert G.digest(d) == REF[name]["d"]
    assert int(tri.sum()) == REF[name]["tri_sum"]


def test_digests_cover_every_case():
    assert set(REF) == set(CASES)


@pytest.mark.parametrize("name", ["pair256", "pair300"])
def test_exact_mode_differs_only_by_the_wrap(name):
    """From WRAP entries on, the exact weights and the reference's differ, on the two vertices that see
    the heavy pair as their opposite edge, by a multiple of WRAP."""
    _, exact, d = oracle(name, False)
    _, ref, _ = oracle(name, True)
    assert G.digest(exact) != REF[name]["tri"] and G.digest(d) == REF[name]["d"]
    diff = exact - ref
    assert np.flatnonzero(diff).tolist() == [2, 3]
    assert np.all(diff % WRAP == 0)


@pytest.mark.skipif(not reflccd.available(), reason="oracle/_ref/ref_lcc_directed_driver is not built")
@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_mode_equals_live_reference(name):
    n, src, dst, oids = CASES[name]
    tri, d = reflccd.run_app(n, src, dst, oids=oids, threads=2)
    _, otri, od = oracle(name, True)
    assert np.array_equal(tri, otri)
    assert np.array_equal(d, od)
