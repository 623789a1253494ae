"""GPU tests of the forward coset transform with the coset folded into twisted twiddles (BJ_NTT_TWIST, get_twist_table and
NttPass.twisted in csrc/ntt.cu): twist on, twist off (the first pass scales every element on load) and the CPU oracle must
agree byte for byte.  Sizes 2^13..2^24 at the benchmark's shapes, coset 7 and the LDE's coset shifts g w_{Ln}^k; one column,
many columns and more than 65535 columns; out-of-place strided LDEs; the generic pass kernel (unaligned base, odd stride);
lanes reading the parent's table cache; the fallback to scaling once the table budget is spent; inputs with non-canonical
values in [p, 2^64).  The dispatch cases check with torch.profiler that the twisted table was built (or not)."""
import contextlib
import ctypes
import os
import time

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

P = O.P
RANDOM_COSET = int(O.random_field(np.random.default_rng(9191), 1)[0]) | 1


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


@pytest.fixture(scope="module")
def on(bj):
    with context(bj, BJ_NTT_TWIST=1) as c:
        yield c


@pytest.fixture(scope="module")
def off(bj):
    with context(bj, BJ_NTT_TWIST=0) as c:
        yield c


def field_input(seed, shape):
    """Canonical random values with about one in seven replaced by a non-canonical value in [p, 2^64)."""
    r = np.random.default_rng(seed)
    a = O.random_field(r, shape)
    mask = r.random(shape) < 1 / 7
    a[mask] = r.integers(P, 2**64, size=int(mask.sum()), dtype=np.uint64)
    return a


def device_input(seed, cols, n):
    """A [cols, n] device batch generated on the GPU (full 64-bit range, plus planted non-canonical values)."""
    import torch
    g = torch.Generator(device="cuda:0")
    g.manual_seed(seed)
    d = torch.randint(-(2**63), 2**63 - 1, (cols, n), dtype=torch.int64, device="cuda:0", generator=g)
    d[:, 3::977] = -(1 << 31)  # 2^64 - 2^31 >= p
    return d


def np64(t):
    return t.detach().cpu().numpy().view(np.uint64)


def check(got, want):
    assert bool((np.asarray(got) < np.uint64(P)).all())
    assert np.array_equal(got, want)


def kernel_names(fn, attempts=3):
    """Names of the CUDA kernels fn() launches, pooled over `attempts` traces (a trace can miss kernels); fn must be
    repeatable."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    names = []
    probe = torch.zeros(1 << 16, dtype=torch.int64, device="cuda:0")
    for _ in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(8):  # probe launches first: a trace can miss the first kernels launched in it
                probe.add_(1)
            torch.cuda.synchronize()
            time.sleep(0.05)
            fn()
            torch.cuda.synchronize()
        names += [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert names, "the profiler recorded no CUDA kernels"
    return names


def has(names, pat):
    return any(pat in n for n in names)


def lde_shift(log_n, log_l, k, next_row=False):
    """The shift of coset k of bj_lde: g w_{Ln}^bitrev_L(k), g = 7, times w_n for the next-row LDE."""
    kr = int(format(k, "0%db" % log_l)[::-1], 2) if log_l else 0
    s = 7 * pow(int(O.omega(log_n + log_l)), kr, P) % P
    return s * int(O.omega(log_n)) % P if next_row else s


# ------------------------------------------------------------------------------ a. bench shapes, twist on / off / oracle -----
@pytest.mark.parametrize("log_n,n_cols", [(13, 1), (13, 512), (14, 3), (16, 64), (17, 2), (20, 128), (21, 64), (22, 32),
                                          (23, 16), (24, 8)])
def test_forward_on_off_oracle(bj, on, off, log_n, n_cols):
    """Forward on coset 7 and on a random coset: twist on == twist off on the whole batch; both == the oracle on columns
    0, 1, middle and last."""
    import torch
    n = 1 << log_n
    d0 = device_input(log_n * 1000 + n_cols, n_cols, n)
    cols = sorted({0, min(1, n_cols - 1), n_cols // 2, n_cols - 1})
    a = np.stack([np64(d0[c]) for c in cols])
    for coset in (7, RANDOM_COSET):
        if log_n >= 22 and coset != 7:
            continue
        d_on, d_off = d0.clone(), d0.clone()
        on.fft_natural_to_bitreversed(d_on, coset)
        off.fft_natural_to_bitreversed(d_off, coset)
        assert torch.equal(d_on, d_off), coset
        del d_off
        check(np.stack([np64(d_on[c]) for c in cols]), O.ntt_n2b(a, coset))
        del d_on
    torch.cuda.empty_cache()


def test_twisted_table_is_used(bj, on, off):
    """A new coset at 2^16: twist on builds a twisted table and no coset-power table; twist off the reverse; a one-pass
    size (2^12) scales on load in both; the inverse never twists."""
    d = device_input(16, 2, 1 << 16)
    small = device_input(12, 2, 1 << 12)

    def fwd(c, t, coset0):
        k = iter(range(100))
        return lambda: c.fft_natural_to_bitreversed(t.clone(), coset0 + next(k))
    names = kernel_names(fwd(on, d, 1000))
    assert has(names, "twist_table_kernel") and not has(names, "pow_table_kernel"), names
    names = kernel_names(fwd(off, d, 2000))
    assert not has(names, "twist_table_kernel") and has(names, "pow_table_kernel"), names
    names = kernel_names(fwd(on, small, 3000))
    assert not has(names, "twist_table_kernel") and has(names, "pow_table_kernel"), names
    k = iter(range(100))
    names = kernel_names(lambda: on.ifft_natural_to_natural(d.clone(), 4000 + next(k)))
    assert not has(names, "twist_table_kernel"), names


# ------------------------------------------------------------------------------ b. more than 65535 columns -----
def test_more_than_65535_columns(bj, on, off):
    import torch
    n_cols, log_n = 65537, 13
    d0 = device_input(65537, n_cols, 1 << log_n)
    cols = [0, 65534, 65535, 65536]
    a = np.stack([np64(d0[c]) for c in cols])
    d_on, d_off = d0.clone(), d0.clone()
    on.fft_natural_to_bitreversed(d_on, 7)
    off.fft_natural_to_bitreversed(d_off, 7)
    assert torch.equal(d_on, d_off)
    check(np.stack([np64(d_on[c]) for c in cols]), O.ntt_n2b(a, 7))
    del d0, d_on, d_off
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------ c. LDE cosets, out of place and strided -----
@pytest.mark.parametrize("log_n,log_l,cols", [(13, 3, 3), (16, 1, 2), (16, 2, 2), (20, 3, 2), (22, 1, 2)])
@pytest.mark.parametrize("from_mono", [False, True])
def test_lde_on_off_oracle(bj, on, off, log_n, log_l, cols, from_mono):
    """bj_lde: each coset g w_{Ln}^k is one forward transform that reads the monomials and writes out of place into columns
    strided by the LDE factor; its next-row variant shifts every coset by w_n."""
    import torch
    a = field_input(log_n * 10 + log_l + from_mono, (cols, 1 << log_n))
    mono = a[:1] if from_mono else O.intt_n2n(a[:1], 1)
    for next_row in (False, True):
        outs = [np64(c.transform_raw_storages_to_lde(bj.to_device(a), 1 << log_l, from_monomials=from_mono, next_row=next_row))
                for c in (on, off)]
        assert np.array_equal(outs[0], outs[1]), next_row
        if log_n <= 16 and not next_row:
            check(outs[0], O.lde(a, log_l, from_monomials=from_mono))
        k = (1 << log_l) - 1  # the last coset of column 0 against the oracle's transform of the monomials on its shift
        check(outs[0][0, k], O.ntt_n2b(mono, lde_shift(log_n, log_l, k, next_row))[0])
    torch.cuda.empty_cache()


@pytest.mark.parametrize("log_n", [13, 16])
def test_lde_coset_shifts(bj, on, log_n):
    """The coset transforms of a factor-8 LDE on the shifts g w_{8n}^bitrev(k), from monomials: each equals the oracle's
    forward NTT of the monomials on that shift."""
    a = field_input(8000 + log_n, (2, 1 << log_n))
    out = np64(on.transform_raw_storages_to_lde(bj.to_device(a), 8, from_monomials=True))
    for k in range(8):
        check(out[:, k], O.ntt_n2b(a, lde_shift(log_n, 3, k)))


# ------------------------------------------------------------------------------ d. generic pass kernel -----
LAYOUTS = {"offset": lambda n: (n, 1), "odd_stride": lambda n: (n + 1, 0)}  # -> (stride, pointer offset in elements)


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("log_n", [13, 16, 17, 20, 22])
def test_generic_kernel(bj, on, off, log_n, layout):
    """8-byte-aligned base pointer or odd column stride: the passes take the generic kernel; the padding is not written."""
    lib = bj.native.lib
    n, cols, fill = 1 << log_n, 2, 0xDEADBEEF
    stride, off_el = LAYOUTS[layout](n)
    a = field_input(log_n * 7 + len(layout), (cols, n))
    buf = np.full(off_el + cols * stride + 3, fill, np.uint64)
    for c in range(cols):
        buf[off_el + c * stride: off_el + c * stride + n] = a[c]
    res = []
    for c in (on, off):
        d = bj.to_device(buf)
        fn = lambda t: lib.bj_ntt_natural_to_bitreversed(c._h, ctypes.c_void_p(t.data_ptr() + 8 * off_el), log_n, cols, stride, 7)  # noqa: E731
        if c is on:
            names = kernel_names(lambda: fn(d.clone()))
            assert has(names, "ntt_pass_kernel") and not has(names, "ntt_pass_v2_kernel"), names
        assert fn(d) == 0, lib.bj_last_error(c._h)
        res.append(bj.to_numpy(d))
    assert np.array_equal(res[0], res[1])
    got = np.stack([res[0][off_el + c * stride: off_el + c * stride + n] for c in range(cols)])
    check(got, O.ntt_n2b(a, 7))
    keep = np.ones(buf.size, bool)
    for c in range(cols):
        keep[off_el + c * stride: off_el + c * stride + n] = False
    assert (res[0][keep] == np.uint64(fill)).all()


def test_generic_kernel_forced_by_v2_off(bj):
    """BJ_NTT_V2=0 on aligned buffers, 2^22: the generic kernel with the twisted table."""
    a = field_input(2222, (2, 1 << 22))
    with context(bj, BJ_NTT_V2=0) as c:
        d = bj.to_device(a)
        c.fft_natural_to_bitreversed(d, 7)
        check(bj.to_numpy(d), O.ntt_n2b(a, 7))


# ------------------------------------------------------------------------------ e. lanes -----
def test_lane_uses_parent_cache(bj):
    """A lane's forward coset transform builds the twisted table into its parent's cache; the parent then reuses it.  Both
    match the oracle."""
    import torch
    a = field_input(4242, (3, 1 << 18))
    coset = RANDOM_COSET ^ 2
    with context(bj) as parent:
        lane = parent.lane()
        d = bj.to_device(a)
        torch.cuda.synchronize()
        lane.fft_natural_to_bitreversed(d, coset)
        lane.synchronize()
        check(bj.to_numpy(d), O.ntt_n2b(a, coset))
        names = kernel_names(lambda: parent.fft_natural_to_bitreversed(bj.to_device(a), coset))
        assert not has(names, "twist_table_kernel"), names
        d = bj.to_device(a)
        parent.fft_natural_to_bitreversed(d, coset)
        check(bj.to_numpy(d), O.ntt_n2b(a, coset))
        lane.close()


# ------------------------------------------------------------------------------ f. budget spent -----
def test_budget_exhausted_falls_back_to_scaling(bj):
    """Six 2^26 twisted tables spend the 3 GiB table budget: a new coset then scales on load (coset-power tables, no
    twisted table) and still matches the oracle and the twist-off context; a coset twisted before keeps its table."""
    import torch
    with context(bj) as c, context(bj, BJ_NTT_TWIST=0) as c_off:
        big = device_input(26, 1, 1 << 26)
        for coset in (3, 5, 6, 10, 11, 12):
            c.fft_natural_to_bitreversed(big, coset)
        a = field_input(2020, (2, 1 << 20))
        k = iter(range(100))
        names = kernel_names(lambda: c.fft_natural_to_bitreversed(bj.to_device(a), 500 + next(k)))
        assert not has(names, "twist_table_kernel") and has(names, "pow_table_kernel"), names
        d, d_off = bj.to_device(a), bj.to_device(a)
        c.fft_natural_to_bitreversed(d, 13)
        c_off.fft_natural_to_bitreversed(d_off, 13)
        assert torch.equal(d, d_off)
        check(bj.to_numpy(d), O.ntt_n2b(a, 13))
        names = kernel_names(lambda: c.fft_natural_to_bitreversed(big, 6))
        assert not has(names, "twist_table_kernel") and not has(names, "pow_table_kernel"), names
        del big
        torch.cuda.empty_cache()
