"""The restatement of iterativelengthbidirectional (oracle/pgq_oracle_bidir.c) against the reference binary's rows.

tests/golden/refb_*.npz come from oracle/_ref/duckdb (tests/golden/make_golden_bidir.py).  The reference reads the key
columns byte by byte, so each golden spells the ids its searches use into the bytes of the columns; the test first
checks that reading, then that the restatement returns the reference's rows on those ids, at its 512 lanes."""
import glob
import os

import numpy as np
import pytest

from oracle import pgq_oracle as orc
from oracle import pgq_oracle_bidir as orb

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "refb_*.npz")))


def test_goldens_present():
    assert len(GOLDEN) >= 17


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[5:-4] for p in GOLDEN])
def test_oracle_matches_reference(path):
    z = np.load(path)
    n = int(z["n"])
    p = len(z["col_src"])
    # what the reference searched: the byte at offset row of each column (iterativelength_bidirectional.cpp:104-110)
    assert np.array_equal(z["col_src"].view(np.uint8)[:p], z["eff_src"])
    assert np.array_equal(z["col_dst"].view(np.uint8)[:p], z["eff_dst"])
    v, e, _ = orc.csr_build(n, z["src"].astype(np.int64), z["dst"].astype(np.int64))
    out, valid, _ = orb.iterativelengthbidirectional(n, v, e, z["eff_src"], z["eff_dst"], z["src_valid"], None, 512)
    assert np.array_equal(valid, z["length_valid"])
    assert np.array_equal(out, z["length"].astype(np.int64))
