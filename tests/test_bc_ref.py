"""The betweenness oracle (oracle/bc_oracle.py, mode "replay") against the
reference's own CPU app: bit for bit against the stored digests of its
one-thread run (tests/golden/ref_bc_outputs.json) on every case of
tests/bc_cases.py, and against the live driver (oracle/_ref/ref_bc_driver,
--threads 1) when it is built."""
import numpy as np
import pytest

from oracle import bc_oracle as BO
from oracle import refbc
from tests import golden_io as G
from tests.bc_cases import as_indices, bc_cases, ref_bc_outputs, source_index

REF = ref_bc_outputs()
CASES = bc_cases()


def replay(name):
    n, src, dst, oids, source = CASES[name]
    s, d = as_indices(n, src, dst, oids)
    return BO.bc(n, s, d, source_index(n, oids, source), "replay")


@pytest.mark.parametrize("name", sorted(CASES))
def test_replay_equals_reference_digests(name):
    c, sigma, depth = replay(name)
    want = REF[name]
    assert want["source"] == CASES[name][4]
    assert G.digest(depth) == want["depth"]
    assert G.digest(sigma) == want["sigma"]
    assert G.digest(c) == want["c"]


def test_reference_digests_cover_every_case():
    assert set(REF) == set(CASES)
    # an absent source reaches nothing; the diamond chain's path counts pass 2^53
    assert REF["rmat12_absent"]["levels"] == 0
    assert REF["diamond_chain40"]["levels"] == 81
    _, sigma, _ = replay("diamond_chain40")
    assert sigma.max() > 2.0 ** 53


@pytest.mark.skipif(not refbc.available(), reason="oracle/_ref/ref_bc_driver is not built")
@pytest.mark.parametrize("name", sorted(CASES))
def test_replay_equals_live_reference(name):
    n, src, dst, oids, source = CASES[name]
    rc, rs, rd = refbc.run_app(n, src, dst, source, oids=oids, threads=1)
    c, sigma, depth = replay(name)
    assert np.array_equal(rd, depth)
    assert np.array_equal(rs.view(np.uint64), sigma.view(np.uint64))
    assert np.array_equal(rc.view(np.uint32), c.view(np.uint32))
