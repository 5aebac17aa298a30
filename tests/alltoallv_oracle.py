"""Brute-force rules of the all-to-all-v in plain Python, for checking the bound plan rules (csrc/kernels/
alltoallv_plan.h) without a GPU.  A count matrix is a list of P rows of P ints: m[p][q] rows from rank p to rank q."""
import random

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
