"""The oracle's restatement of iterativelengthbidirectional on the CPU: the properties its contract states."""
import numpy as np

from duckpgq_extension_b200 import datagen
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_bidir as orb


def test_undirected_graph_gives_iterativelength():
    n, s, d = datagen.rmat_edges(9, seed=1)
    s, d = np.concatenate([s, d]), np.concatenate([d, s])
    v, e, _ = orc.csr_build(n, s, d)
    rng = np.random.default_rng(2)
    src, dst = rng.integers(0, n, 1500), rng.integers(0, n, 1500)
    src[::9] = dst[::9]
    sv = (rng.random(1500) > 0.1).astype(np.uint8)
    out, valid, st = orb.iterativelengthbidirectional(n, v, e, src, dst, sv)
    eo, ev, _ = orc.iterativelength(n, v, e, src, dst, sv, 512)
    assert np.array_equal(valid, ev) and np.array_equal(out, eo)
    assert st.batches == 3


def test_answer_depends_on_the_batch():
    n = 10
    v, e, _ = orc.csr_build(n, np.array([1, 2, 3, 4]), np.array([0, 3, 4, 5]))
    out, valid, st = orb.iterativelengthbidirectional(n, v, e, np.array([0]), np.array([1]))
    assert valid[0] == 0 and (st.batches, st.iterations, st.edges_traversed) == (1, 1, 0)
    out, valid, st = orb.iterativelengthbidirectional(n, v, e, np.array([2, 0]), np.array([9, 1]))
    assert list(valid) == [0, 1] and out[1] == 2
    # at 64 lanes the two rows fall into different batches once 64 rows sit between them
    src, dst = np.array([2] * 64 + [0]), np.array([9] * 64 + [1])
    out, valid, st = orb.iterativelengthbidirectional(n, v, e, src, dst, lanes=64)
    assert valid[-1] == 0 and st.batches == 2
    out, valid, st = orb.iterativelengthbidirectional(n, v, e, src, dst, lanes=128)
    assert valid[-1] == 1 and out[-1] == 2 and st.batches == 1


def test_null_destination_and_trivial_rows_take_no_lane():
    # on 0 -> 1 -> 2 the destination side of (0, 2) has no out-edge: its first level adds nothing and the row is NULL
    n = 4
    v, e, _ = orc.csr_build(n, np.array([0, 1]), np.array([1, 2]))
    out, valid, st = orb.iterativelengthbidirectional(n, v, e, np.array([0, 3, 0]), np.array([2, 3, 99]),
                                                      dst_valid=np.array([1, 1, 0]))
    assert list(valid) == [0, 1, 0] and list(out) == [-1, 0, -1] and st.iterations == 2
