"""CPU check of the forward coset transform with the coset folded into the twiddles (get_twist_table / NttPass.twisted in
era_boojum_b200/csrc/ntt.cu, transcribed in tools/ntt_model.py) against the oracle's scaled coset NTT, for every plan
shape and tile setting test_ntt_model.py enumerates."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import ntt_model as M  # noqa: E402
from oracle import oracle as O  # noqa: E402

P = M.P
RANDOM_COSET = int(O.random_field(np.random.default_rng(4711), 1)[0]) | 1


@pytest.mark.parametrize("log_n", [1, 4, 9])
@pytest.mark.parametrize("coset", [7, RANDOM_COSET])
def test_twist_table_squares_chain(log_n, coset):
    """tw[1]^2 = c^n, and the twiddles of a group's two children square to its own and to its negation (round r splits
    X^d - z into X^(d/2) -+ s): tw[2^(r+1) + 2G]^2 = tw[2^r + G], tw[2^(r+1) + 2G + 1]^2 = -tw[2^r + G]."""
    tw = M.twist_table(log_n, coset)
    assert len(tw) == 1 << log_n
    assert tw[1] * tw[1] % P == pow(coset, 1 << log_n, P)
    for r in range(log_n - 1):
        for g in range(1 << r):
            even, odd = tw[(2 << r) + 2 * g], tw[(2 << r) + 2 * g + 1]
            assert even * even % P == tw[(1 << r) + g]
            assert (odd * odd + tw[(1 << r) + g]) % P == 0


@pytest.mark.parametrize("m", [4, 5, 7, 10, 13, 14])
@pytest.mark.parametrize("coset", [7, RANDOM_COSET])
def test_twisted_model_matches_oracle(m, coset):
    a = O.random_field(np.random.default_rng(m + 17), 1 << m)
    a[::7] |= np.uint64(0xFFFFFFFF00000000)  # some non-canonical inputs in [p, 2^64)
    got, _ = M.transform(a, coset, False, twist=True)
    assert np.array_equal(got, O.ntt_n2b(a, coset))


@pytest.mark.parametrize("m,maxe,pass1_w", [(13, 8, -1), (14, 8, -1), (13, 9, -1), (14, 10, 0), (13, 13, 1), (14, 12, 3),
                                            (14, 14, 5), (13, 11, 4)])
def test_twisted_model_matches_oracle_tile_settings(m, maxe, pass1_w):
    a = O.random_field(np.random.default_rng(200 + m + maxe), 1 << m)
    a[::5] |= np.uint64(0xFFFFFFFF00000000)
    got, plan = M.transform(a, 7, False, maxe, pass1_w, twist=True)
    assert plan == M.make_plan(m, False, maxe, pass1_w)
    assert np.array_equal(got, O.ntt_n2b(a, 7)), plan


def test_twist_is_forward_coset_only():
    """No coset, or the inverse: the model takes the plain table whatever `twist` says."""
    a = O.random_field(np.random.default_rng(5), 1 << 6)
    assert np.array_equal(M.transform(a, 1, False, twist=True)[0], O.ntt_n2b(a, 1))
    assert np.array_equal(M.transform(a, 7, True, twist=True)[0], O.intt_n2n(a, 7))
