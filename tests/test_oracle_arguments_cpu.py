"""The C oracle's copy-permutation, lookup and Horner restatements (oracle/oracle.c) against the Python-int ones
(oracle/stage2.py, oracle/lookup.py) at small sizes.  The Python oracles are tied to the reference through the CPU
prover; the GPU tests at production sizes (tests/test_gpu_argument_paths.py) compare against the C ones, which are fast
enough there.  Inputs include non-canonical representatives in [p, 2^64)."""
import numpy as np
import pytest

from oracle import lookup as LK
from oracle import oracle as O
from oracle import replay
from oracle import stage2 as S

P = O.P


def rng(seed):
    return np.random.default_rng(seed)


def lazy(r, a, frac=0.25):
    """a with p added to a seeded subset of the cells below 2^32 - 1 (same field elements, non-canonical bits)"""
    a = np.array(a, dtype=np.uint64)
    mask = (r.random(a.shape) < frac) & (a < np.uint64(2**32 - 1))
    a[mask] += np.uint64(P)
    return a


def wide(r, shape):
    """uniform over all 64-bit words: about 2^-32 of them are in [p, 2^64), so plant some explicitly"""
    a = r.integers(0, 2**64, size=shape, dtype=np.uint64)
    mask = r.random(shape) < 0.2
    a[mask] = r.integers(P, 2**64, size=int(mask.sum()), dtype=np.uint64)
    return a


def satisfying_copy_permutation(r, n_cols, log_n):
    """values and sigma columns whose copy constraints hold: cells in cycles of three share one (small) value"""
    n = 1 << log_n
    ks = S.non_residues_for_copy_permutation(n, n_cols)
    w_n = replay.omega(log_n)
    vals = r.integers(0, 2**31, size=(n_cols, n), dtype=np.uint64)
    sig = np.array([[ks[j] * pow(w_n, i, P) % P for i in range(n)] for j in range(n_cols)], dtype=np.uint64)
    cells = [(j, i) for j in range(n_cols) for i in range(n)]
    perm = r.permutation(len(cells))
    for g in range(0, len(cells) - 2, 3):
        cyc = [cells[perm[g + t]] for t in range(3)]
        v = vals[cyc[0]]
        for (j, i), (j2, i2) in zip(cyc, cyc[1:] + cyc[:1]):
            vals[j, i] = v
            sig[j, i] = ks[j2] * pow(w_n, i2, P) % P
    # sigma is below 2^32 - 1 only where it names a row-0 cell (k_j is a small integer): all of those become non-canonical
    return lazy(r, vals), lazy(r, sig, 1.0), ks


def e2(r):
    return tuple(int(x) for x in O.random_field(r, 2))


def pairs(c0, c1):
    return [(int(a), int(b)) for a, b in zip(c0, c1)]


# ------------------------------------------------------------------------------------------- stage 2 -----
@pytest.mark.parametrize("n_cols,chunk,log_n", [(5, 1, 4), (7, 3, 5), (5, 8, 6), (6, 6, 3), (9, 4, 6), (1, 1, 2)])
def test_cp_stage2_matches_python(n_cols, chunk, log_n):
    r = rng(10 * n_cols + chunk + log_n)
    vals, sig, ks = satisfying_copy_permutation(r, n_cols, log_n)
    assert (vals >= np.uint64(P)).any() and (sig >= np.uint64(P)).any()
    beta, gamma = e2(r), e2(r)
    wz, wp = S.partial_products([list(map(int, c)) for c in vals], [list(map(int, c)) for c in sig], beta, gamma, chunk)
    z0, z1, partials, grand = O.cp_stage2(list(vals), list(sig), ks, beta, gamma, chunk)
    assert grand == (1, 0)
    assert pairs(z0, z1) == wz
    assert len(partials) == len(wp) == (n_cols + chunk - 1) // chunk - 1
    for got, want in zip(partials, wp):
        assert pairs(got[0], got[1]) == want


def test_cp_stage2_grand_product_of_a_broken_copy():
    r = rng(3)
    vals, sig, ks = satisfying_copy_permutation(r, 4, 5)
    vals[2, 31] = (int(vals[2, 31]) + 1) % P
    *_, grand = O.cp_stage2(list(vals), list(sig), ks, e2(r), e2(r), 3)
    assert grand != (1, 0)


# ------------------------------------------------------------------------- copy-permutation quotient -----
@pytest.mark.parametrize("n_cols,chunk,log_n,log_lde,log_q", [
    (5, 2, 4, 3, 0),    # Q = 1
    (5, 2, 4, 3, 1),    # Q = 2 < L
    (7, 3, 3, 3, 3),    # Q = L = 8, last chunk partial
    (4, 8, 4, 2, 2),    # one chunk
    (6, 1, 3, 1, 1),    # chunk 1, Q = L = 2
])
def test_cp_quotient_and_division_match_python(n_cols, chunk, log_n, log_lde, log_q):
    """The relation is pointwise, so random LDE columns are enough (non-canonical ones included)."""
    r = rng(100 * n_cols + 10 * log_lde + log_q)
    n_chunks = (n_cols + chunk - 1) // chunk
    full = 1 << (log_n + log_lde)
    npts = 1 << (log_n + log_q)
    v, s = wide(r, (n_cols, full)), wide(r, (n_cols, full))
    z = wide(r, (2, full))
    part = wide(r, (max(n_chunks - 1, 1), 2, full))[:n_chunks - 1]
    beta, gamma = e2(r), e2(r)
    alphas = [e2(r) for _ in range(n_chunks + 1)]
    init = wide(r, (2, npts))
    ks = S.non_residues_for_copy_permutation(1 << log_n, n_cols)
    q0, q1 = O.cp_quotient(list(v), list(s), ks, (z[0], z[1]), [(p[0], p[1]) for p in part], beta, gamma, alphas,
                           log_n, log_lde, log_q, chunk, init[0], init[1])
    for t in range(npts):
        term = S.quotient_copy_permutation_point(t, log_n, log_lde, v, s, (z[0], z[1]), [(p[0], p[1]) for p in part],
                                                 beta, gamma, alphas, chunk)
        assert (int(q0[t]), int(q1[t])) == ((int(init[0, t]) + term[0]) % P, (int(init[1, t]) + term[1]) % P), t
    d0, d1 = O.divide_by_vanishing(lazy(r, q0), lazy(r, q1), log_n, log_q)
    for t in range(npts):
        vi = S.vanishing_inverse(log_n, log_q, t >> log_n)
        assert (int(d0[t]), int(d1[t])) == (int(q0[t]) * vi % P, int(q1[t]) * vi % P), t


# -------------------------------------------------------------------------------------------- lookup -----
@pytest.mark.parametrize("n_sub,width,with_id", [(1, 1, False), (8, 3, True), (8, 4, True), (32, 7, True), (32, 8, False),
                                                 (1, 8, False), (8, 1, True), (32, 4, False)])
def test_lookup_polys_and_quotient_match_python(n_sub, width, with_id):
    r = rng(1000 * n_sub + 10 * width + with_id)
    log_n, log_q = 4, 1
    n, npts = 1 << log_n, 1 << (log_n + log_q)
    n_tab = width + int(with_id)
    cols = wide(r, (n_sub * width, n))
    tid = wide(r, n) if with_id else None
    tabs = wide(r, (n_tab, n))
    mult = wide(r, n)
    beta, gamma = e2(r), e2(r)
    got = O.lookup_polys(list(cols), width, tid, list(tabs), mult, beta, gamma)
    wA, wB = LK.lookup_polys(list(cols), width, tid, list(tabs), mult, beta, gamma)
    for i in range(n_sub):
        assert pairs(got[i, 0], got[i, 1]) == wA[i], i
    assert pairs(got[n_sub, 0], got[n_sub, 1]) == wB

    L_cols = wide(r, (n_sub * width, npts))
    L_tid = wide(r, npts) if with_id else None
    L_tabs, L_mult = wide(r, (n_tab, npts)), wide(r, npts)
    L_a, L_b = wide(r, (n_sub, 2, npts)), wide(r, (2, npts))
    alphas = [e2(r) for _ in range(n_sub + 1)]
    init = wide(r, (2, npts))
    a_ldes = [(L_a[i, 0], L_a[i, 1]) for i in range(n_sub)]
    q0, q1 = O.lookup_quotient(list(L_cols), width, L_tid, list(L_tabs), L_mult, a_ldes, (L_b[0], L_b[1]), beta, gamma, alphas,
                               init[0], init[1])
    for t in range(npts):
        term = LK.quotient_lookup_point(t, list(L_cols), width, L_tid, list(L_tabs), L_mult, a_ldes, (L_b[0], L_b[1]), beta,
                                        gamma, alphas)
        assert (int(q0[t]), int(q1[t])) == ((int(init[0, t]) + term[0]) % P, (int(init[1, t]) + term[1]) % P), t


# ------------------------------------------------------------------------------------------- Horner ------
@pytest.mark.parametrize("log_n", [0, 1, 5, 6])
def test_horner_ext_matches_python(log_n):
    r = rng(log_n)
    mono = wide(r, (3, 1 << log_n))
    for at in (e2(r), (0, 0), (int(O.omega(4)), 0), (P - 1, P - 1)):
        got = O.horner_ext(mono, at)
        for c in range(3):
            assert (int(got[c, 0]), int(got[c, 1])) == S.horner_ext(mono[c], at)


def test_horner_on_intt_is_the_polynomial_through_the_values():
    """orc_intt_n2n then Horner at omega^i gives back the i-th value: the pair is the barycentric reference."""
    r = rng(77)
    log_n = 5
    vals = wide(r, (2, 1 << log_n))
    mono = O.intt_n2n(vals)
    for i in (0, 1, 17, 31):
        got = O.horner_ext(mono, (int(O.pow_(O.omega(log_n), i)), 0))
        assert [int(x) for x in got[:, 0]] == [int(v) % P for v in vals[:, i]]
        assert not got[:, 1].any()
