"""The core decomposition / k-core oracle (oracle/core_oracle.py) against the
reference's own CPU apps: bit for bit against the stored digests
(tests/golden/ref_core_outputs.json) on every case of tests/core_cases.py, and
against the live driver (oracle/_ref/ref_core_driver) when it is built."""
import numpy as np
import pytest

from oracle import core_oracle as CO
from oracle import refcore
from tests import golden_io as G
from tests.core_cases import as_indices, core_cases, ref_core_outputs

REF = ref_core_outputs()
CASES = core_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference_digests(name):
    n, src, dst, oids, _ = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    want = REF[name]
    core, _ = CO.core_decomposition(n, s, d)
    assert G.digest(core) == want["core"]
    assert (int(core.max()) if n else 0) == want["max_core"]
    for k, dg in want["kcore"].items():
        assert G.digest(CO.kcore(n, s, d, int(k))) == dg, k


def test_reference_digests_cover_the_issue_inputs():
    assert set(REF) == set(CASES)
    assert sorted(int(k) for k in REF["p2p31"]["kcore"]) == [0, 3, 6, 7]
    assert REF["p2p31"]["max_core"] == 6


@pytest.mark.skipif(not refcore.available(), reason="oracle/_ref/ref_core_driver is not built")
@pytest.mark.parametrize("name", sorted(core_cases(big=False)))
def test_oracle_equals_live_reference(name):
    n, src, dst, oids, ks = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    core, _ = CO.core_decomposition(n, s, d)
    assert np.array_equal(refcore.run_app("core_decomposition", n, src, dst, oids=oids), core)
    for k in ks + [int(core.max()) + 1]:
        assert np.array_equal(refcore.run_app("kcore", n, src, dst, k=k, oids=oids), CO.kcore(n, s, d, k)), k
