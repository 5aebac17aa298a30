"""The all-to-all-v plan rules as bound from csrc/kernels/alltoallv_plan.h (the ones the kernel, bin/alltoall --cpu and
the emulated device run) against the brute force of tests/alltoallv_oracle.py: the verdict and its rule order, the
packed send and receive offsets, on random matrices at 1-16 ranks and on the edge cases of the capacities."""
import random

import pytest

from tests import alltoallv_oracle as oracle

INT64_MAX = (1 << 63) - 1


@pytest.fixture(scope="module")
def C(native):
    return native


def _verdict(C, m, send_cap, recv_cap):
    return C.alltoallv_verdict(oracle.flat(m), len(m), send_cap, recv_cap)


@pytest.mark.parametrize("P", range(1, 17))
def test_random_matrices_against_brute_force(C, P):
    rng = random.Random(P)
    for trial in range(60):
        hi = rng.choice([1, 3, 10, 1000])
        m = oracle.random_matrix(rng, P, hi)
        if trial % 5 == 0:
            m[rng.randrange(P)][rng.randrange(P)] = -rng.randint(1, 5)
        sums = [sum(r) for r in m] + [sum(m[p][q] for p in range(P)) for q in range(P)]
        for send_cap, recv_cap in ((max(sums + [1]), max(sums + [1])), (rng.randint(1, 2 * hi * P), rng.randint(1, 2 * hi * P))):
            assert _verdict(C, m, send_cap, recv_cap) == oracle.verdict(m, send_cap, recv_cap), (m, send_cap, recv_cap)
        if oracle.verdict(m, INT64_MAX, INT64_MAX) == 0:
            for p in range(P):
                for q in range(P):
                    assert C.alltoallv_send_offset(oracle.flat(m), P, p, q) == oracle.send_offset(m, p, q)
                    assert C.alltoallv_recv_offset(oracle.flat(m), P, p, q) == oracle.recv_offset(m, p, q)


@pytest.mark.parametrize("P", [1, 2, 3, 5, 8, 16])
def test_segments_tile_the_buffers(C, P):
    """The receive segments of every rank tile [0, total) in rank order with no gap or overlap, and the send segments
    of an accepted matrix stay inside the send capacity."""
    rng = random.Random(100 + P)
    for _ in range(20):
        m = oracle.random_matrix(rng, P, 9)
        cap = max([sum(r) for r in m] + [sum(m[p][q] for p in range(P)) for q in range(P)] + [1])
        assert _verdict(C, m, cap, cap) == 0
        f = oracle.flat(m)
        for r in range(P):
            at = 0
            for p in range(P):
                assert C.alltoallv_recv_offset(f, P, p, r) == at
                at += m[p][r]
            assert at <= cap
            covered = set()
            for q in range(P):
                lo = C.alltoallv_send_offset(f, P, r, q)
                seg = set(range(lo, lo + m[r][q]))
                assert not (seg & covered) and all(0 <= x < cap for x in seg)
                covered |= seg


def test_edge_cases(C):
    P, cap = 4, 12
    assert _verdict(C, [[0] * P for _ in range(P)], 1, 1) == 0                      # zeros
    at = [[0, 3, 0, 0] for _ in range(P)]                                             # a column exactly at capacity
    assert _verdict(C, at, cap, cap) == 0
    at[2][1] += 1                                                                     # one row over it
    assert _verdict(C, at, cap, cap) == oracle.RECV_CAPACITY
    one = [[0] * P for _ in range(P)]
    one[3][0] = cap + 1                                                               # a single count above capacity
    assert _verdict(C, one, cap, 10 * cap) == oracle.SEND_CAPACITY
    both = [row[:] for row in one]
    both[0][2] = -1                                                                   # negatives with overflows: rule 1
    both[1] = [INT64_MAX] * P
    assert _verdict(C, both, cap, cap) == oracle.NEGATIVE
    huge = [[INT64_MAX] * P for _ in range(P)]                                        # no int64 overflow in the sums
    assert _verdict(C, huge, INT64_MAX, INT64_MAX) == oracle.SEND_CAPACITY
    cols = [[INT64_MAX // P] * P for _ in range(P)]
    assert _verdict(C, cols, INT64_MAX, INT64_MAX // 2) == oracle.RECV_CAPACITY


def test_every_rank_computes_the_same_verdict(C):
    """Ranks differ only in the matrix they read, which is the same for all: the verdict is a function of the matrix
    and the capacities only, whatever order the rows arrived in."""
    rng = random.Random(7)
    for _ in range(50):
        P = rng.randint(2, 16)
        m = oracle.random_matrix(rng, P, 5)
        if rng.random() < 0.3:
            m[rng.randrange(P)][rng.randrange(P)] = -1
        caps = (rng.randint(1, 5 * P), rng.randint(1, 5 * P))
        verdicts = {_verdict(C, [row[:] for row in m], *caps) for _ in range(P)}
        assert len(verdicts) == 1 and verdicts.pop() == oracle.verdict(m, *caps)


def test_bad_matrix_shape_is_refused(C):
    with pytest.raises(Exception, match="world x world"):
        C.alltoallv_verdict([1, 2, 3], 2, 4, 4)
    with pytest.raises(Exception, match="world x world"):
        C.alltoallv_verdict([0] * 289, 17, 4, 4)
