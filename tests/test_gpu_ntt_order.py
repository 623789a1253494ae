"""GPU tests of the NTT tile passes' column-fastest work order (BJ_NTT_COL_FASTEST, launch_pass in csrc/ntt.cu): one CTA per
(tile, column) on a one-dimensional grid, the same tile of every column back to back.  Every setting (the default rule,
front passes only, last passes only, both) must give results bit-identical to the tile-fastest order (0) and to the CPU
oracle: forward with no coset, coset 7 and a random coset (full and two-level coset-power tables), the inverse's front passes,
in place (the transforms) and out of place into strided columns (LDE), one column, more than 65535 columns, and inputs
with non-canonical values."""
import contextlib
import os

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

P = O.P
RANDOM_COSET = int(O.random_field(np.random.default_rng(777), 1)[0]) | 1
ORDERS = [-1, 1, 2, 3]


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


@contextlib.contextmanager
def context(bj, **env):
    """A context created with the given BJ_* environment switches (restored right after creation), closed at exit."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        c = bj.Context.on_current_stream(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v
    try:
        yield c
    finally:
        c.synchronize()
        c.close()


def field_input(seed, shape):
    """Canonical random values with about one in seven replaced by a non-canonical value in [p, 2^64)."""
    r = np.random.default_rng(seed)
    a = O.random_field(r, shape)
    mask = r.random(shape) < 1 / 7
    a[mask] = r.integers(P, 2**64, size=int(mask.sum()), dtype=np.uint64)
    return a


def run(bj, env, a, coset, inverse):
    with context(bj, **env) as c:
        d = bj.to_device(a)
        if inverse:
            c.ifft_natural_to_natural(d, coset)
        else:
            c.fft_natural_to_bitreversed(d, coset)
        c.synchronize()
        return bj.to_numpy(d)


@pytest.mark.parametrize("full_pow", [1, 0])
@pytest.mark.parametrize("log_n,cols", [(12, 5), (13, 1), (16, 3), (17, 2), (20, 2), (22, 2), (23, 1)])
def test_forward_orders_bit_identical(bj, log_n, cols, full_pow):
    """Sizes with one and two passes, the 2^22 and 2^23 front passes whose coset table exceeds the L2 set-aside."""
    for coset in (1, 7, RANDOM_COSET):
        a = field_input(log_n * 31 + cols + coset % 13, (cols, 1 << log_n))
        want = run(bj, {"BJ_NTT_COL_FASTEST": 0, "BJ_NTT_FULL_POW": full_pow}, a, coset, False)
        if (cols << log_n) <= 1 << 17:
            assert np.array_equal(want, O.ntt_n2b(a, coset))
        for order in ORDERS:
            got = run(bj, {"BJ_NTT_COL_FASTEST": order, "BJ_NTT_FULL_POW": full_pow}, a, coset, False)
            assert bool((got < np.uint64(P)).all())
            assert np.array_equal(got, want), (order, coset)


@pytest.mark.parametrize("log_n,cols", [(16, 3), (21, 2)])
def test_inverse_front_passes(bj, log_n, cols):
    a = field_input(log_n + cols, (cols, 1 << log_n))
    want = run(bj, {"BJ_NTT_COL_FASTEST": 0}, a, 7, True)
    if log_n <= 16:
        assert np.array_equal(want, O.intt_n2n(a, 7))
    for order in ORDERS:
        assert np.array_equal(run(bj, {"BJ_NTT_COL_FASTEST": order}, a, 7, True), want)


def test_more_than_65535_columns(bj):
    cols, log_n = 70001, 5
    a = field_input(99, (cols, 1 << log_n))
    want = run(bj, {"BJ_NTT_COL_FASTEST": 0}, a, 7, False)
    sub = np.r_[0:3, 65534:65538, cols - 3:cols]
    assert np.array_equal(want[sub], O.ntt_n2b(a[sub], 7))
    for order in ORDERS:
        assert np.array_equal(run(bj, {"BJ_NTT_COL_FASTEST": order}, a, 7, False), want)


@pytest.mark.parametrize("log_n,log_lde,cols", [(12, 1, 5), (16, 3, 2), (22, 1, 2)])
def test_lde_out_of_place_strided(bj, log_n, log_lde, cols):
    """bj_lde: every coset transform reads the monomials and writes out of place into columns strided by the LDE factor."""
    a = field_input(log_n + log_lde, (cols, 1 << log_n))
    outs = []
    for order in [0] + ORDERS:
        with context(bj, BJ_NTT_COL_FASTEST=order) as c:
            outs.append(bj.to_numpy(c.transform_raw_storages_to_lde(bj.to_device(a), 1 << log_lde)))
    for o in outs[1:]:
        assert np.array_equal(o, outs[0])
    if log_n <= 16:
        assert np.array_equal(outs[0], O.lde(a, log_lde))
