"""The maths of a split domain shard on the CPU oracle: row block p of coset j (rows [p n / B, (p + 1) n / B) in the
coset's bit-reversed row order) is the coset sigma * <w_{n/B}>, sigma = 7 w_{nL}^{bitrev_L(j)} w_n^{bitrev_s(p)}, and on it
f(x) = sum_{k < n/B} b_k x^k with b_k = sum_{m < B} sigma^(m n / B) a_{k + m n / B}.  So a fold of the monomials followed by
one size-n/B coset NTT on sigma gives the row block of the LDE - what bj_lde does on a split shard."""
import numpy as np
import pytest

from oracle import oracle as O


def _bitrev(x, bits):
    return int(format(x, "0%db" % bits)[::-1], 2) if bits else 0


def _unit_shift(j, p, log_n, log_l, s):
    c = O.mul(7, O.pow_(O.omega(log_n + log_l), _bitrev(j, log_l)))
    return O.mul(c, O.pow_(O.omega(log_n), _bitrev(p, s)))


def _fold(mono, sigma, nb, blocks):
    """b_k = sum_m sigma^(m nb) a_{k + m nb}"""
    sb = O.pow_(sigma, nb)
    out = np.zeros((mono.shape[0], nb), np.uint64)
    for c in range(mono.shape[0]):
        for k in range(nb):
            acc, pw = 0, 1
            for m in range(blocks):
                acc = O.add(acc, O.mul(int(mono[c, k + m * nb]), pw))
                pw = O.mul(pw, sb)
            out[c, k] = acc
    return out


@pytest.mark.parametrize("s", [1, 2, 3])
@pytest.mark.parametrize("log_l", [1, 2])
def test_fold_then_coset_ntt_is_the_row_block(s, log_l):
    log_n, cols = 7, 3
    n, B = 1 << log_n, 1 << s
    nb = n // B
    rng = np.random.default_rng(100 * s + log_l)
    vals = O.random_field(rng, (cols, n))
    mono = O.intt_n2n(vals)
    want = O.lde(vals, log_l)
    for j in range(1 << log_l):
        for p in range(B):
            sigma = _unit_shift(j, p, log_n, log_l, s)
            got = O.ntt_n2b(_fold(mono, sigma, nb, B), sigma)
            assert np.array_equal(got, want[:, j, p * nb:(p + 1) * nb]), (j, p)


@pytest.mark.parametrize("s", [1, 2, 3])
def test_next_row_block_is_the_shift_by_omega(s):
    """z(w x) on a row block: the unit LDE on sigma * w_n, in the same row order, equals the unsharded LDE read at
    position bitrev(bitrev(i) + 1) of the same coset."""
    log_n, log_l = 6, 1
    n, B = 1 << log_n, 1 << s
    nb = n // B
    rng = np.random.default_rng(7 + s)
    vals = O.random_field(rng, (2, n))
    mono = O.intt_n2n(vals)
    full = O.lde(vals, log_l)
    nxt = [_bitrev((_bitrev(i, log_n) + 1) % n, log_n) for i in range(n)]
    for j in range(1 << log_l):
        shifted = full[:, j, nxt]
        for p in range(B):
            sigma = O.mul(_unit_shift(j, p, log_n, log_l, s), O.omega(log_n))
            got = O.ntt_n2b(_fold(mono, sigma, nb, B), sigma)
            assert np.array_equal(got, shifted[:, p * nb:(p + 1) * nb]), (j, p)
