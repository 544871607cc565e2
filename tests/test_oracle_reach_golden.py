"""The restatement of reachability (oracle/pgq_oracle_reach.c) against the reference binary's rows.

tests/golden/refr_*.npz come from oracle/_ref/duckdb (tests/golden/make_golden_reach.py), for both traversals.  The
reference reads the key columns byte by byte, so each golden spells the ids its searches use into the bytes of the
columns; the test first checks that reading, then that the restatement -- with the reference's own batch start, NULL
restart included -- returns the reference's row wherever the source and the destination are valid."""
import glob
import os

import numpy as np
import pytest

from oracle import pgq_oracle as orc
from oracle import pgq_oracle_reach as orr

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "refr_*.npz")))


def test_goldens_present():
    assert len(GOLDEN) >= 12


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[5:-4] for p in GOLDEN])
def test_oracle_matches_reference(path, variant):
    z = np.load(path)
    n = int(z["n"])
    p = len(z["col_src"])
    # what the reference searched: the byte at offset row of each column (reachability.cpp:26,242)
    assert np.array_equal(z["col_src"].view(np.uint8)[:p], z["eff_src"])
    assert np.array_equal(z["col_dst"].view(np.uint8)[:p], z["eff_dst"])
    v, e, _ = orc.csr_build(n, z["src"].astype(np.int64), z["dst"].astype(np.int64))
    ok = (z["src_valid"] & z["dst_valid"]).astype(bool)
    out, written, _ = orr.reachability(n, v, e, z["eff_src"], z["eff_dst"], z["src_valid"], z["dst_valid"],
                                       is_variant=bool(variant), restart=True)
    assert z[f"reach{variant}_valid"][ok].all() and written[ok].all()
    assert np.array_equal(out[ok], z[f"reach{variant}"][ok]), np.nonzero(out[ok] != z[f"reach{variant}"][ok])[0][:10]
    # the plain traversal's answers do not depend on the batches: the defined batch start gives them too
    if not variant:
        d_out, d_written, _ = orr.reachability(n, v, e, z["eff_src"], z["eff_dst"], z["src_valid"], z["dst_valid"])
        assert np.array_equal(d_written.astype(bool), ok) and np.array_equal(d_out[ok], z["reach0"][ok])


def test_stale_visit_list_confirmed_by_the_reference():
    """With is_variant, the batch the NULL restart starts runs over the first batch's visit_list: the reference itself
    answers (0, 5) false in the last row, and true with the plain traversal."""
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "refr_stale_visit_list.npz"))
    assert (z["eff_src"][-1], z["eff_dst"][-1]) == (0, 5)
    assert z["reach0"][-1] == 1 and z["reach1"][-1] == 0
    ok = (z["src_valid"] & z["dst_valid"]).astype(bool)
    assert np.array_equal(z["reach0"][ok][:-1], z["reach1"][ok][:-1])
