"""CPU check of the NTT planner / tile / stage / twiddle-index arithmetic used by the CUDA kernel
(tools/ntt_model.py transcribes era_boojum_b200/csrc/ntt.cu) against the oracle."""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import ntt_model as M  # noqa: E402
from oracle import oracle as O  # noqa: E402


@pytest.mark.parametrize("m", [4, 5, 7, 10, 13, 14])
@pytest.mark.parametrize("coset", [1, 7])
def test_model_matches_oracle(m, coset):
    a = O.random_field(np.random.default_rng(m), 1 << m)
    f, _ = M.transform(a, coset, False)
    assert np.array_equal(f, O.ntt_n2b(a, coset))
    g, _ = M.transform(a, coset, True)
    assert np.array_equal(g, O.intt_n2n(a, coset))


# non-default tile settings (BJ_NTT_MAX_TILE_LOG, BJ_NTT_PASS1_W): 3-pass plans at 2^13 / 2^14, narrow and wide tiles
@pytest.mark.parametrize("m,maxe,pass1_w", [(13, 8, -1), (14, 8, -1), (13, 9, -1), (14, 10, 0), (13, 13, 1), (14, 12, 3),
                                            (14, 14, 5), (13, 11, 4)])
def test_model_matches_oracle_tile_settings(m, maxe, pass1_w):
    a = O.random_field(np.random.default_rng(100 + m + maxe), 1 << m)
    a[::5] |= np.uint64(0xFFFFFFFF00000000)  # some non-canonical inputs in [p, 2^64)
    for inv in (False, True):
        got, plan = M.transform(a, 7, inv, maxe, pass1_w)
        assert plan == M.make_plan(m, inv, maxe, pass1_w)
        assert np.array_equal(got, O.intt_n2n(a, 7) if inv else O.ntt_n2b(a, 7)), (inv, plan)


def _cuda_plan_capacity():
    """Number of passes ntt.cu's `struct Plan` can hold (its array length, a literal or a named constant)."""
    src = open(os.path.join(ROOT, "era_boojum_b200", "csrc", "ntt.cu")).read()
    n = re.search(r"struct Plan \{[^}]*?\bint t\[(\w+)\];", src).group(1)
    if not n.isdigit():
        n = re.search(r"constexpr int %s = (\d+);" % n, src).group(1)
    return int(n)


def test_plans_cover_all_rounds():
    """Every plan of every allowed tile setting (BJ_NTT_MAX_TILE_LOG is clamped to 8..14, BJ_NTT_PASS1_W < 0 means
    automatic) covers all rounds with legal tiles and fits the CUDA planner's Plan."""
    cap = _cuda_plan_capacity()
    for maxe in range(8, 15):
        for pass1_w in (-1, 0, 1, 2, 3, 4, 5):
            for m in range(4, 33):
                for inv in (False, True):
                    plan = M.make_plan(m, inv, maxe, pass1_w)
                    where = (maxe, pass1_w, m, inv, plan)
                    assert len(plan) <= cap, where
                    assert sum(t for t, _ in plan) == m, where
                    r0 = 0
                    for i, (t, w) in enumerate(plan):
                        last = i == len(plan) - 1
                        assert 4 <= t + w <= max(12, maxe), where
                        assert w >= 0, where
                        if not (inv and last):
                            assert w <= m - r0 - t, where
                        else:
                            assert w <= r0, where
                        r0 += t
    assert M.NTT_MAX_PASSES == cap
