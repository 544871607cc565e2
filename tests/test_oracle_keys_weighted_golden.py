"""The position rule of the weighted key builds, pinned against the reference binary on the CPU.

tests/golden/refkw_*.npz hold what the unmodified reference made of key columns with a weight column (the CSR CTE with
k.w as create_csr_edge's last argument): get_csr_v / get_csr_e / get_csr_w, csr_get_w_type and cheapest_path_length.
The key restatement (oracle/pgq_oracle_keys) gives the CSR and the edge row of every position; the weight of a position
is then w[edge row], the weight of the row that became it.  That must equal get_csr_w bit for bit, -0.0 and NaNs
included, once both are in the same order within each source row (DuckDB's join hands a vertex's rows over in its own
order)."""
import os

import numpy as np
import pytest

from oracle import pgq_oracle as orc
from oracle import pgq_oracle_keys as ork

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = sorted(f[6:-4] for f in os.listdir(GOLDEN) if f.startswith("refkw_") and f.endswith(".npz"))


def load(name):
    z = np.load(os.path.join(GOLDEN, f"refkw_{name}.npz"))
    return {k: z[k] for k in z.files}


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64) if a.dtype.kind == "f" else a.astype(np.int64)


def per_vertex_sorted(v, e, w, n):
    """(target, weight bits) of every position, in a canonical order within each source row."""
    row = np.repeat(np.arange(n), np.diff(np.asarray(v[:n + 1], dtype=np.int64)))
    wb = bits(w)
    order = np.lexsort((wb, np.asarray(e), row))
    return np.asarray(e)[order], wb[order]


def test_fixtures_cover_the_layouts():
    assert len(NAMES) >= 6
    kinds = {int(load(nm)["w_type"]) for nm in NAMES}
    assert kinds == {1, 2}
    joined_dup = unjoined_null = False
    for nm in NAMES:
        g = load(nm)
        unjoined_null |= bool(np.any(g["w_valid"] == 0))
        joined_dup |= g["csr_e"].shape[0] > int(np.count_nonzero(g["src_valid"]))
    assert joined_dup and unjoined_null
    f = np.concatenate([load(nm)["w"] for nm in NAMES if load(nm)["w"].dtype.kind == "f"])
    assert np.any(np.isnan(f)) and np.any((f == 0) & np.signbit(f)) and np.any(f < 0)
    i = np.concatenate([load(nm)["w"] for nm in NAMES if load(nm)["w"].dtype.kind != "f"])
    assert {np.iinfo(np.int64).max, np.iinfo(np.int64).min} <= set(i.tolist())


@pytest.mark.parametrize("name", NAMES)
def test_weight_of_a_position_is_the_weight_of_its_edge_row(name):
    g = load(name)
    n = g["vkey"].shape[0]
    v, e, ids = ork.csr_build_keys(g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    assert np.array_equal(v, g["csr_v"])
    assert int(g["w_type"]) == (2 if g["w"].dtype.kind == "f" else 1)
    assert np.all(g["w_valid"][ids] == 1)  # a joined edge never has a NULL weight
    w = g["w"][ids]
    for a, b in zip(per_vertex_sorted(v, e, w, n), per_vertex_sorted(g["csr_v"], g["csr_e"], g["csr_w"], n)):
        assert np.array_equal(a, b)  # bit for bit


@pytest.mark.parametrize("name", NAMES)
def test_cheapest_path_length_restatement_on_the_key_csr(name):
    """The Bellman-Ford restatement on the key build's CSR answers as the reference did."""
    g = load(name)
    n = g["vkey"].shape[0]
    v, e, ids = ork.csr_build_keys(g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    cost, valid = orc.cheapest_path_length(n, v, e, g["w"][ids], g["psrc"], g["pdst"])
    assert np.array_equal(valid, g["cost_valid"])
    assert np.array_equal(bits(cost[valid == 1]), bits(g["cost"][valid == 1]))
