"""Brute-force rules of the all-to-all-v in plain Python, for checking the bound plan rules (csrc/kernels/
alltoallv_plan.h) without a GPU.  A count matrix is a list of P rows of P ints: m[p][q] rows from rank p to rank q."""
import random

import torch

NEGATIVE, SEND_CAPACITY, RECV_CAPACITY = 1, 2, 3


def verdict(m, send_cap, recv_cap):
    """0 if the matrix is accepted, else the lowest broken rule: a negative count, a count or row sum above the send
    capacity, a column sum above the receive capacity (Python ints: no overflow to worry about)."""
    P = len(m)
    cells = [c for row in m for c in row]
    if any(c < 0 for c in cells):
        return NEGATIVE
    if any(c > send_cap for c in cells) or any(sum(row) > send_cap for row in m):
        return SEND_CAPACITY
    if any(sum(m[p][q] for p in range(P)) > recv_cap for q in range(P)):
        return RECV_CAPACITY
    return 0


def send_offset(m, p, q):
    return sum(m[p][:q])


def recv_offset(m, p, r):
    return sum(m[j][r] for j in range(p))


def flat(m):
    return [c for row in m for c in row]


def random_matrix(rng: random.Random, P, hi, zeros=0.2):
    return [[0 if rng.random() < zeros else rng.randint(0, hi) for _ in range(P)] for _ in range(P)]


# The count matrices the GPU tests launch: random with zeros, all zero, a single pair, local only, one column exactly at
# the receive capacity, and one hot column.
PATTERNS = ["random", "zero", "single", "local", "column-at-capacity", "skewed"]


def counts_for(pattern, P, mean, cap, launch, gen):
    """A P x P matrix (list of lists) of ``pattern`` that fits capacities of `cap` rows; a new one for every launch
    (``gen`` is a CPU torch.Generator)."""
    ri = lambda hi: int(torch.randint(0, hi + 1, (1,), generator=gen))
    m = [[0] * P for _ in range(P)]
    if pattern == "random":
        m = [[ri(2 * mean) for _ in range(P)] for _ in range(P)]
        for _ in range(max(1, P // 2)):
            m[ri(P - 1)][ri(P - 1)] = 0
    elif pattern == "single":
        m[launch % P][(launch * 7 + 1) % P] = 1 + ri(cap - 1)
    elif pattern == "local":
        for p in range(P):
            m[p][p] = 1 + ri(2 * mean)
    elif pattern == "column-at-capacity":
        c = launch % P
        for p in range(P):
            for q in range(P):
                m[p][q] = ri(mean // P)
        for p in range(P):
            m[p][c] = cap // P + (cap % P if p == P - 1 else 0)
    elif pattern == "skewed":
        hot = launch % P
        for p in range(P):
            for q in range(P):
                m[p][q] = 2 * mean if q == hot else ri(mean // P)
    return m
