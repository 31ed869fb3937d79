"""Symmetric random views (SWIM_TOPO_SYMMETRIC) from the host generator, against an independent NumPy statement of the
definition (include/swim.h, DESIGN.md 2.3): the union of degree / 2 random Hamiltonian cycles, cycle c visiting the nodes
in the order of (word i & 3 of Philox (c, i >> 2, 11, 0), i). No device needed."""
import numpy as np
import pytest

from swim_b200 import _abi as A
from swim_b200._lib import SwimError
from swim_b200.sim import generate_topology

NM = A.NO_MEMBER


def symmetric_numpy(n, cap, degree, seed):
    from oracle.oracle import philox
    key = (seed & 0xFFFFFFFF, seed >> 32)
    pred, succ = np.empty((degree // 2, n), np.int64), np.empty((degree // 2, n), np.int64)
    for c in range(degree // 2):
        blocks = np.array([philox((c, g, 11, 0), key) for g in range((n + 3) // 4)], dtype=np.uint64).reshape(-1)
        keys = blocks[:n]  # node i: block i >> 2, word i & 3
        order = np.lexsort((np.arange(n), keys))  # by key, ties by id
        pred[c, order] = np.roll(order, 1)
        succ[c, order] = np.roll(order, -1)
    out = np.full((n, cap), NM, dtype=np.uint32)
    for i in range(n):
        row = np.unique(np.concatenate([pred[:, i], succ[:, i]]))
        out[i, :len(row)] = row
    return out


CASES = [(3, 32, 2, 1), (5, 32, 4, 7), (64, 32, 32, 3), (64, 64, 16, 2 ** 40 + 5), (1001, 32, 32, 11), (1001, 128, 100, 12),
         (1001, 256, 256, 13), (4099, 32, 32, 0x5EED0006), (4099, 64, 10, 99), (33, 32, 32, 4), (257, 256, 256, 8)]


@pytest.mark.parametrize("n,cap,deg,seed", CASES)
def test_host_generator_equals_numpy_statement(n, cap, deg, seed):
    got = generate_topology("symmetric", n, cap, deg, seed=seed)
    assert np.array_equal(got, symmetric_numpy(n, cap, deg, seed))


@pytest.mark.parametrize("n,cap,deg", [(3, 32, 2), (64, 32, 32), (1001, 256, 256), (4099, 32, 32), (20000, 64, 48)])
def test_properties(n, cap, deg):
    nbr = generate_topology("symmetric", n, cap, deg, seed=21)
    present = nbr != NM
    cnt = present.sum(axis=1)
    assert cnt.min() >= 2 and cnt.max() <= deg
    assert np.all(present[:, :-1] >= present[:, 1:])  # vacancies last
    rows = nbr.astype(np.int64)
    assert np.all(np.where(present[:, 1:], np.diff(rows, axis=1) > 0, True))  # ascending, each id once
    i, s = np.nonzero(present)
    j = rows[i, s]
    assert np.all(j != i) and j.max() < n
    edges = set(zip(i.tolist(), j.tolist()))
    assert all((b, a) in edges for a, b in edges)  # symmetric
    if n > 4 * deg:
        assert np.mean(cnt == deg) > 0.5  # a row has fewer than degree members only where cycles repeat a neighbour


def test_same_seed_same_view_other_seed_other_view():
    a, b = generate_topology("symmetric", 3000, 32, 32, seed=9), generate_topology("symmetric", 3000, 32, 32, seed=9)
    assert np.array_equal(a, b)
    assert not np.array_equal(a, generate_topology("symmetric", 3000, 32, 32, seed=10))
    assert not np.array_equal(a, generate_topology("symmetric", 3000, 32, 32, seed=9 + 2 ** 32))


@pytest.mark.parametrize("n,cap,deg,code", [(100, 32, 7, A.EINVAL), (100, 32, 31, A.EINVAL), (100, 32, 0, A.EINVAL),
                                            (2, 32, 2, A.EINVAL), (1, 32, 0, A.EINVAL), (100, 32, 34, A.ECAP),
                                            (300, 256, 258, A.ECAP), (5, 32, 6, A.ECAP)])
def test_error_codes(n, cap, deg, code):
    with pytest.raises(SwimError) as e:
        generate_topology("symmetric", n, cap, deg, seed=1)
    assert e.value.code == code
