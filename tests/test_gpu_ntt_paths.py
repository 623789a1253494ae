"""GPU tests of the NTT family (forward, inverse, LDE, bit reversal, host-buffer pipeline) on the paths the default-layout
parity tests in test_gpu_parity.py do not reach: the generic pass kernel (8-byte-aligned pointers, odd strides,
BJ_NTT_V2=0), non-default tile settings, the two-level coset-power tables, column chunking, batches of more than 65535
columns, the host-buffer ring and coset-sharded LDEs.

Every case compares the GPU result bit for bit with the CPU oracle (oracle/liboracle.so) on seeded inputs that include
non-canonical values in [p, 2^64), and checks that outputs are canonical.  The dispatch tests also check, with
torch.profiler, that the kernel they target is the one that ran, so that a change of the dispatch rule cannot silently
turn them into more tests of the default path."""
import contextlib
import ctypes
import os
import re
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import ntt_model as M  # noqa: E402

pytestmark = pytest.mark.gpu

P = O.P
GENERIC = "ntt_pass_kernel"
# tile shapes (t, w) with a specialised kernel (the instantiation menu of csrc/ntt_v2.cuh)
V2_MENU = {(t, 0) for t in range(4, 15)} | {(11, 2), (8, 3), (9, 3), (10, 3), (11, 3), (8, 4), (9, 4), (10, 4),
                                            (6, 5), (7, 5), (8, 5), (9, 5)}


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


@pytest.fixture(scope="module")
def lib(bj):
    from era_boojum_b200 import native
    return native.lib


@pytest.fixture(scope="module")
def ctx(bj):
    c = bj.Context.on_current_stream(0)
    yield c
    c.synchronize()
    c.close()


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


def rng(seed):
    return np.random.default_rng(seed)


def field_input(seed, shape):
    """Canonical random values with about one in seven replaced by a non-canonical value in [p, 2^64)."""
    r = rng(seed)
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
    d[:, 5::1031] = -(1 << 31)  # 2^64 - 2^31 >= p
    return d


def canonical(a):
    return bool((np.asarray(a) < np.uint64(P)).all())


def check(got, want):
    assert canonical(got)
    assert np.array_equal(got, want)


def call(bj, ctx, fn, *args):
    st = fn(ctx._h, *args)
    assert st == 0, "status %d: %s" % (st, bj.native.lib.bj_last_error(ctx._h).decode())


def ptr(t, offset=0):
    return ctypes.c_void_p(t.data_ptr() + 8 * offset)


_probe = {}


@pytest.fixture(scope="module", autouse=True)
def _close_probe():
    yield
    if _probe:
        _probe.pop("ctx").close()
        _probe.clear()


def _trace_once(fn):
    import time
    import torch
    from torch.profiler import ProfilerActivity, profile
    import era_boojum_b200 as bj
    if not _probe:
        _probe["ctx"] = bj.Context.on_current_stream(0)
        _probe["buf"] = torch.zeros(16, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(8):  # probe launches first: a trace can miss the first kernels launched in it
            _probe["ctx"].bitreverse_enumeration_inplace(_probe["buf"])
        torch.cuda.synchronize()
        time.sleep(0.05)
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "bitreverse_kernel" not in e.name]


def kernels_run(make_fn, attempts=3):
    """Names of the CUDA kernels launched by make_fn(k)() for k < attempts, recorded with torch.profiler.

    A trace can miss some of the kernels the library launches, so the call is traced `attempts` times and the names of
    all traces are returned together.  make_fn(k) must be repeatable: the same dispatch for every k, on throwaway data."""
    names = []
    for k in range(attempts):
        names += _trace_once(make_fn(k))
    assert names, "the profiler recorded no CUDA kernels"
    return names


def has(names, pat):
    return any(pat in n for n in names)


def v2_shapes(names):
    """(t, w, kind) of the specialised pass kernels that ran (demangled or mangled names)."""
    out = set()
    for n in names:
        if "ntt_pass_v2_kernel" not in n:
            continue
        m = re.search(r"ntt_pass_v2_kernel\w*<(\d+), (\d+), (\d+)>", n) or re.search(r"ntt_pass_v2_kernel\w*ILi(\d+)ELi(\d+)ELi(\d+)E", n)
        assert m, n
        out.add(tuple(int(x) for x in m.groups()))
    return out


def expected_passes(m, inverse, maxe=13, pass1_w=-1):
    """(t, w, kind) of the passes of a transform on aligned buffers that take a specialised kernel, and whether one of
    them takes the generic kernel.  The specialised one-column tiles (w = 0) serve contiguous last passes only."""
    if m < 4:
        return set(), False
    plan = M.make_plan(m, inverse, maxe, pass1_w)
    v2, generic = set(), False
    for i, (t, w) in enumerate(plan):
        last = i == len(plan) - 1
        if (t, w) in V2_MENU and (w > 0 or last):
            v2.add((t, w, 1 if inverse and last else 0))
        else:
            generic = True
    return v2, generic


def padded(a, stride, offset, fill):
    """Columns of a at `stride` elements from each other, starting `offset` elements into a filled buffer."""
    cols, n = a.shape
    buf = np.full(offset + cols * stride + 3, fill, np.uint64)
    for c in range(cols):
        buf[offset + c * stride: offset + c * stride + n] = a[c]
    return buf


def unpad(buf, cols, n, stride, offset):
    return np.stack([buf[offset + c * stride: offset + c * stride + n] for c in range(cols)])


def padding_intact(buf, cols, n, stride, offset, fill):
    keep = np.ones(buf.size, bool)
    for c in range(cols):
        keep[offset + c * stride: offset + c * stride + n] = False
    return bool((buf[keep] == np.uint64(fill)).all())


# ------------------------------------------------------------------------------ a. generic pass kernel -----
LAYOUTS = {"offset": lambda n: (n, 1), "odd_stride": lambda n: (n + 1, 0)}   # -> (stride, pointer offset in elements)
SIZES = [4, 8, 12, 13, 16, 17, 20, 21, 22, 24]
RANDOM_COSET = int(O.random_field(rng(4242), 1)[0]) | 1


def _cosets(log_n, layout, inverse):
    # every coset at the smaller sizes; one per case above 2^17, where the oracle dominates the run time
    cs = [1, 7, RANDOM_COSET]
    return cs if log_n <= 17 else [cs[(log_n + len(layout) + inverse) % 3]]


def traced(op, d):
    """Kernel names of op(t) on a fresh copy t of d (the checked run is made separately, without the profiler)."""
    def make(k):
        t = d.clone()
        return lambda: op(t)
    return kernels_run(make)


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("log_n", SIZES)
def test_generic_kernel_unaligned_layouts(bj, ctx, lib, log_n, layout, inverse):
    """8-byte-aligned base pointer or odd column stride: every pass takes the generic kernel, padding is not written."""
    n, cols, fill = 1 << log_n, 2, 0xDEADBEEF
    stride, off = LAYOUTS[layout](n)
    fn = lib.bj_intt_natural_to_natural if inverse else lib.bj_ntt_natural_to_bitreversed
    for coset in _cosets(log_n, layout, inverse):
        a = field_input(log_n * 100 + coset % 97 + inverse, (cols, n))
        d = bj.to_device(padded(a, stride, off, fill))
        names = traced(lambda t: call(bj, ctx, fn, ptr(t, off), log_n, cols, stride, coset), d)
        assert has(names, GENERIC) and not has(names, "ntt_pass_v2_kernel"), names
        call(bj, ctx, fn, ptr(d, off), log_n, cols, stride, coset)
        buf = bj.to_numpy(d)
        check(unpad(buf, cols, n, stride, off), O.intt_n2n(a, coset) if inverse else O.ntt_n2b(a, coset))
        assert padding_intact(buf, cols, n, stride, off, fill)


def test_generic_kernel_three_pass_forward_2pow25(bj, ctx, lib):
    """2^25 forward, plan (6,5),(6,5),(13,0), through the generic kernel on an 8-byte-aligned buffer."""
    log_n, cols = 25, 2
    n = 1 << log_n
    assert len(M.make_plan(log_n, False)) == 3
    a = field_input(2525, (cols, n))
    d = bj.to_device(padded(a, n, 1, 0))
    fwd = lambda t: call(bj, ctx, lib.bj_ntt_natural_to_bitreversed, ptr(t, 1), log_n, cols, n, 7)  # noqa: E731
    names = traced(fwd, d)
    assert has(names, GENERIC) and not has(names, "ntt_pass_v2_kernel"), names
    fwd(d)
    check(unpad(bj.to_numpy(d), cols, n, n, 1), O.ntt_n2b(a, 7))


@pytest.mark.parametrize("log_n", [10, 16])
@pytest.mark.parametrize("log_l", [1, 3])
@pytest.mark.parametrize("from_mono", [False, True])
@pytest.mark.parametrize("layout", ["in_odd_stride", "in_offset_out_offset"])
def test_generic_kernel_lde(bj, ctx, lib, log_n, log_l, from_mono, layout):
    """bj_lde from an odd-strided input, or from an offset input into an offset output (the coset transforms then take
    the generic kernel too).  Kernels mix where a pass stays in aligned memory: a multi-pass inverse ends in the library's
    scratch, and a multi-pass forward into an aligned output runs its later passes in place there."""
    import torch
    n, cols, fill = 1 << log_n, 3, 77
    stride, in_off, out_off = (n + 1, 0, 0) if layout == "in_odd_stride" else (n, 1, 1)
    a = field_input(log_n * 10 + log_l + from_mono, (cols, n))
    d_in = bj.to_device(padded(a, stride, in_off, fill))
    before = d_in.clone()
    out = torch.full((out_off + cols * (n << log_l) + 2,), fill, dtype=torch.int64, device="cuda:0")
    lde = lambda o: call(bj, ctx, lib.bj_lde, ptr(d_in, in_off), stride, ptr(o, out_off), log_n, log_l, cols, int(from_mono))  # noqa: E731
    names = traced(lde, out)
    assert has(names, GENERIC), names
    multi = len(M.make_plan(log_n, True)) > 1 and len(M.make_plan(log_n, False)) > 1
    v2_expected = (multi and not from_mono) or (layout == "in_odd_stride" and (multi or not from_mono))
    assert has(names, "ntt_pass_v2_kernel") == v2_expected, names
    lde(out)
    got = bj.to_numpy(out)
    check(got[out_off: out_off + cols * (n << log_l)].reshape(cols, 1 << log_l, n), O.lde(a, log_l, from_monomials=from_mono))
    assert (got[:out_off] == fill).all() and (got[out_off + cols * (n << log_l):] == fill).all()
    assert torch.equal(d_in, before)


def test_generic_kernel_odd_stride_inverse_mixes_kernels(bj, ctx, lib):
    """A multi-pass inverse whose ping-pong ends in the stride-n scratch (an LDE from odd-strided values): the passes that
    touch the odd-strided columns take the generic kernel, the pass between the aligned scratch buffers the specialised."""
    import torch
    log_n, cols = 16, 2
    n = 1 << log_n
    a = field_input(1616, (cols, n))
    d_in = bj.to_device(padded(a, n + 1, 0, 5))
    out = torch.empty((cols, 2, n), dtype=torch.int64, device="cuda:0")
    lde = lambda o: call(bj, ctx, lib.bj_lde, ptr(d_in), n + 1, ptr(o), log_n, 1, cols, 0)  # noqa: E731
    names = traced(lde, out)
    plan = M.make_plan(log_n, True)
    assert len(plan) == 2
    assert has(names, GENERIC), names
    t, w = plan[-1]
    assert (t, w, 1) in v2_shapes(names), names  # the transposing last pass, scratch -> scratch
    lde(out)
    check(bj.to_numpy(out), O.lde(a, 1))


def _transform(c, inverse, coset):
    return lambda t: c.ifft_natural_to_natural(t, coset) if inverse else c.fft_natural_to_bitreversed(t, coset)


@pytest.mark.parametrize("log_n", [12, 16, 22])
def test_generic_kernel_forced_by_v2_off(bj, log_n):
    """BJ_NTT_V2=0 on aligned buffers: forward, inverse and LDE through the generic kernel only."""
    cols = 2
    a = field_input(3000 + log_n, (cols, 1 << log_n))
    with context(bj, BJ_NTT_V2=0) as c:
        for inverse in (False, True):
            d = bj.to_device(a)
            names = traced(_transform(c, inverse, 7), d)
            assert has(names, GENERIC) and not has(names, "ntt_pass_v2_kernel"), names
            _transform(c, inverse, 7)(d)
            check(bj.to_numpy(d), O.intt_n2n(a, 7) if inverse else O.ntt_n2b(a, 7))
        if log_n <= 16:
            out = c.transform_raw_storages_to_lde(bj.to_device(a), 4)
            check(bj.to_numpy(out), O.lde(a, 2))


# ------------------------------------------------------------------------------ b. tile tunables -----
def _differing_size(maxe, pass1_w, sizes=(13, 16, 20, 22)):
    for m in sizes:
        if all(M.make_plan(m, inv, maxe, pass1_w) != M.make_plan(m, inv) for inv in (False, True)):
            return m
    return sizes[0]  # BJ_NTT_PASS1_W=5 is the automatic choice at every size


TUNABLES = [(e, -1) for e in (8, 9, 10, 11, 12, 14)] + [(13, w) for w in range(6)]


def _check_dispatch(names, m, inverse, maxe, pass1_w):
    v2, generic = expected_passes(m, inverse, maxe, pass1_w)
    assert v2_shapes(names) == v2, (names, M.make_plan(m, inverse, maxe, pass1_w))
    assert has(names, GENERIC) == generic, names


@pytest.mark.parametrize("maxe,pass1_w", TUNABLES)
def test_tile_tunables(bj, maxe, pass1_w):
    """BJ_NTT_MAX_TILE_LOG / BJ_NTT_PASS1_W at a size where the plan differs from the default: the passes that ran are
    the ones the planner model predicts, and forward, inverse and LDE match the oracle."""
    m = _differing_size(maxe, pass1_w)
    cols = 2
    a = field_input(maxe * 100 + pass1_w + m, (cols, 1 << m))
    with context(bj, BJ_NTT_MAX_TILE_LOG=maxe, BJ_NTT_PASS1_W=pass1_w) as c:
        for inverse in (False, True):
            d = bj.to_device(a)
            _check_dispatch(traced(_transform(c, inverse, 7), d), m, inverse, maxe, pass1_w)
            _transform(c, inverse, 7)(d)
            check(bj.to_numpy(d), O.intt_n2n(a, 7) if inverse else O.ntt_n2b(a, 7))
        lm = min(m, 16)
        out = c.transform_raw_storages_to_lde(bj.to_device(a[:, : 1 << lm]), 4)
        check(bj.to_numpy(out), O.lde(a[:, : 1 << lm], 2))


@pytest.mark.parametrize("log_n,inverse", [(25, True), (27, False)])
def test_tile_tunables_five_pass_plans(bj, log_n, inverse):
    """BJ_NTT_MAX_TILE_LOG=8: the five-pass plans (inverse of 2^25, forward of 2^27), one column each."""
    import torch
    assert len(M.make_plan(log_n, inverse, 8)) == 5
    a = field_input(log_n, (1, 1 << log_n))
    with context(bj, BJ_NTT_MAX_TILE_LOG=8) as c:
        d = bj.to_device(a)
        _check_dispatch(traced(_transform(c, inverse, 7), d), log_n, inverse, 8, -1)
        _transform(c, inverse, 7)(d)
        got = bj.to_numpy(d)
        del d
        torch.cuda.empty_cache()
    check(got, O.intt_n2n(a, 7) if inverse else O.ntt_n2b(a, 7))


# ------------------------------------------------------------------------------ c. coset-power tables -----
def _tables_built(names):
    """(two-level tables built, expanded table built) in a traced call."""
    return has(names, "pow_table_kernel"), has(names, "pow_full_kernel")


def _tables_for_new_coset(c, d, inverse, coset0):
    """Which tables a coset this context has not seen gets (each trace attempt uses another unseen coset)."""
    def make(k):
        t = d.clone()
        return lambda: _transform(c, inverse, coset0 + k)(t)
    return _tables_built(kernels_run(make))


@pytest.mark.parametrize("log_n", [13, 16, 20, 22, 24])
def test_two_level_pow_tables(bj, log_n):
    """BJ_NTT_FULL_POW=0: coset powers come from the lo * hi tables (SCALE_POW) in the multi-pass forward's first pass
    and the inverse's transposed last pass."""
    cols = 2 if log_n <= 22 else 1
    a = field_input(5000 + log_n, (cols, 1 << log_n))
    with context(bj, BJ_NTT_FULL_POW=0) as c:
        for inverse, coset in ((False, 7), (True, 7), (False, RANDOM_COSET), (True, RANDOM_COSET)):
            if log_n >= 22 and coset != 7:
                continue
            d = bj.to_device(a)
            assert _tables_for_new_coset(c, d, inverse, 1000 + coset) == (True, False)
            _transform(c, inverse, coset)(d)
            check(bj.to_numpy(d), O.intt_n2n(a, coset) if inverse else O.ntt_n2b(a, coset))
        if log_n in (16, 20):
            out = c.transform_raw_storages_to_lde(bj.to_device(a[:1]), 8)
            check(bj.to_numpy(out), O.lde(a[:1], 3))


def test_pow_table_budget_exhausted(bj):
    """A fresh default context: six 2^26 cosets spend the 3 GiB expanded-table budget; later cosets get only the
    two-level tables, while a coset cached before keeps its expanded table."""
    import torch
    log_big = 26
    fill = [3, 5, 6, 10, 11, 12]
    with context(bj) as c:
        d = device_input(26, 1, 1 << log_big)
        for coset in fill:  # 6 x 512 MiB of expanded tables: the whole budget
            c.fft_natural_to_bitreversed(d, coset)
        for log_n in (20, 22):
            a = field_input(log_n + 60, (2, 1 << log_n))
            for inverse, coset in ((False, 13), (True, 14)):
                dd = bj.to_device(a)
                assert _tables_for_new_coset(c, dd, inverse, 100 + coset) == (True, False)
                _transform(c, inverse, coset)(dd)
                check(bj.to_numpy(dd), O.intt_n2n(a, coset) if inverse else O.ntt_n2b(a, coset))
        # a coset cached while the budget lasted: no table is rebuilt, the expanded one is used
        assert _tables_built(traced(_transform(c, False, fill[2]), d)) == (False, False)
        a = field_input(2626, (1, 1 << log_big))
        d.copy_(bj.to_device(a))
        c.fft_natural_to_bitreversed(d, fill[2])
        got = bj.to_numpy(d)
        del d
        torch.cuda.empty_cache()
    check(got, O.ntt_n2b(a, fill[2]))


def test_pow_table_cache_flush(bj):
    """70 distinct cosets at 2^10 (the table cache holds 64, then drops everything), each checked; then the first cosets
    again: their tables are rebuilt, and cached after that."""
    log_n = 10
    cosets = [int(x) | 1 for x in O.random_field(rng(64), 70)]
    a = field_input(6464, (2, 1 << log_n))
    with context(bj) as c:
        for coset in cosets:
            d = bj.to_device(a)
            c.fft_natural_to_bitreversed(d, coset)
            check(bj.to_numpy(d), O.ntt_n2b(a, coset))
        d = bj.to_device(a)

        def first_cosets(k):
            t = d.clone()
            return lambda: c.fft_natural_to_bitreversed(t, cosets[k])
        assert _tables_built(kernels_run(first_cosets)) == (True, True)
        c.fft_natural_to_bitreversed(d, cosets[0])
        check(bj.to_numpy(d), O.ntt_n2b(a, cosets[0]))
        d = bj.to_device(a)  # and now it is cached
        assert _tables_built(traced(_transform(c, False, cosets[0]), d)) == (False, False)
        c.fft_natural_to_bitreversed(d, cosets[0])
        check(bj.to_numpy(d), O.ntt_n2b(a, cosets[0]))


# ------------------------------------------------------------------------------ d. batch shapes -----
def _sample(d, cols):
    return np.stack([bj_np(d[c]) for c in cols])


def bj_np(t):
    return t.detach().cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("log_n,n_cols", [(20, 128), (22, 32), (24, 8)])
def test_forward_bench_batches(bj, ctx, log_n, n_cols):
    """The benchmark's forward shapes (1 GiB each), coset 7; columns 0, 1, middle, last."""
    d = device_input(log_n, n_cols, 1 << log_n)
    cols = [0, 1, n_cols // 2, n_cols - 1]
    a = _sample(d, cols)
    ctx.fft_natural_to_bitreversed(d, 7)
    check(_sample(d, cols), O.ntt_n2b(a, 7))


def test_inverse_two_chunks(bj, ctx):
    """2^20 x 130 columns: the inverse's scratch holds 128 columns, so the batch runs in two chunks."""
    d = device_input(130, 130, 1 << 20)
    cols = [0, 127, 128, 129]
    a = _sample(d, cols)
    ctx.ifft_natural_to_natural(d, 7)
    check(_sample(d, cols), O.intt_n2n(a, 7))


@pytest.mark.parametrize("log_l", [1, 2])
@pytest.mark.parametrize("from_mono", [False, True])
def test_lde_two_chunks(bj, ctx, log_l, from_mono):
    """2^20 x 66 columns: bj_lde works in chunks of 64 columns; columns 63, 64, 65 on every coset, input untouched."""
    d = device_input(66 + log_l, 66, 1 << 20)
    before = d.clone()
    cols = [63, 64, 65]
    out = ctx.transform_raw_storages_to_lde(d, 1 << log_l, from_monomials=from_mono)
    import torch
    assert torch.equal(d, before)
    got = np.stack([bj_np(out[c]) for c in cols])
    check(got, O.lde(_sample(d, cols), log_l, from_monomials=from_mono))


def test_lde_production_shape_three_chunks(bj, ctx):
    """The prover's committed columns: 155 columns at 2^20 on 8 cosets (about 11 GiB), in chunks of 64, 64 and 27."""
    import torch
    d = device_input(155, 155, 1 << 20)
    cols = [0, 64 + 17, 128, 154]
    a = _sample(d, cols)
    out = ctx.transform_raw_storages_to_lde(d, 8)
    got = np.stack([bj_np(out[c]) for c in cols])
    del out, d
    torch.cuda.empty_cache()
    check(got, O.lde(a, 3))


# ------------------------------------------------------------------------------ e. more than 65535 columns -----
@pytest.mark.parametrize("log_n", [4, 10])
def test_more_than_65535_columns(bj, ctx, log_n):
    """65537 columns (the kernel grids' column dimension is at most 65535): forward, inverse, LDE and bit reversal."""
    import torch
    n_cols, n = 65537, 1 << log_n
    cols = [0, 65534, 65535, 65536]
    d0 = device_input(65537 + log_n, n_cols, n)
    a = _sample(d0, cols)
    d = d0.clone()
    ctx.fft_natural_to_bitreversed(d, 7)
    check(_sample(d, cols), O.ntt_n2b(a, 7))
    d.copy_(d0)
    ctx.ifft_natural_to_natural(d, 7)
    check(_sample(d, cols), O.intt_n2n(a, 7))
    d.copy_(d0)
    ctx.bitreverse_enumeration_inplace(d)
    assert np.array_equal(_sample(d, cols), O.bitreverse(a))
    del d
    out = ctx.transform_raw_storages_to_lde(d0, 2)
    check(np.stack([bj_np(out[c]) for c in cols]), O.lde(a, 1))
    del out, d0
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------ f. host-buffer pipeline -----
@contextlib.contextmanager
def pinned(lib, count):
    p = ctypes.c_void_p()
    assert lib.bj_alloc_host_pinned(8 * count, ctypes.byref(p)) == 0
    try:
        yield np.ctypeslib.as_array((ctypes.c_uint64 * count).from_address(p.value))
    finally:
        lib.bj_free_host_pinned(p)


def _host_call(bj, c, lib, h, log_n, n_cols, coset, inverse):
    fn = lib.bj_intt_natural_to_natural_host if inverse else lib.bj_ntt_natural_to_bitreversed_host
    call(bj, c, fn, h.ctypes.data_as(ctypes.c_void_p), log_n, n_cols, coset)


def test_host_pipeline_small_chunks(bj, lib):
    """BJ_NTT_CHUNK_MB=1: 11 columns of 2^16 run as 6 chunks (the 3-slot ring wraps twice, the last chunk is partial),
    pinned and pageable, forward and inverse; then a 2^18 call grows the ring and a 2^16 call reuses it; then a call right
    behind an asynchronous device transform on the same context."""
    with context(bj, BJ_NTT_CHUNK_MB=1) as c:
        for log_n, n_cols in ((16, 11), (18, 5), (16, 11)):
            n = 1 << log_n
            for inverse in (False, True):
                a = field_input(log_n * 7 + inverse, (n_cols, n))
                want = O.intt_n2n(a, 7) if inverse else O.ntt_n2b(a, 7)
                with pinned(lib, n_cols * n) as h:
                    h[:] = a.reshape(-1)
                    _host_call(bj, c, lib, h, log_n, n_cols, 7, inverse)
                    check(h.reshape(n_cols, n), want)
                h = a.copy()  # pageable
                _host_call(bj, c, lib, h, log_n, n_cols, 7, inverse)
                check(h, want)
        d = device_input(99, 4, 1 << 22)
        da = _sample(d, [0, 3])
        c.fft_natural_to_bitreversed(d, 7)  # queued, not waited for
        a = field_input(1111, (11, 1 << 16))
        h = a.copy()
        _host_call(bj, c, lib, h, 16, 11, 7, True)
        check(h, O.intt_n2n(a, 7))
        check(_sample(d, [0, 3]), O.ntt_n2b(da, 7))


@pytest.mark.parametrize("log_n,n_cols", [(24, 8), (20, 128)])
def test_host_pipeline_bench_shapes(bj, ctx, lib, log_n, n_cols):
    """The benchmark's host-buffer shapes at the default chunk size: 2^24 x 8 in pinned memory, 2^20 x 128 pageable."""
    import torch
    n = 1 << log_n
    cols = [0, n_cols // 2 + 1, n_cols - 1]
    if log_n == 24:
        t = torch.empty((n_cols, n), dtype=torch.int64, pin_memory=True)
        h = t.numpy().view(np.uint64)
    else:
        h = np.empty((n_cols, n), np.uint64)
    h[:] = bj_np(device_input(log_n + n_cols, n_cols, n))
    a = h[cols].copy()
    _host_call(bj, ctx, lib, h, log_n, n_cols, 7, False)
    check(h[cols], O.ntt_n2b(a, 7))


# ------------------------------------------------------------------------------ g. coset-sharded LDE -----
@pytest.mark.parametrize("from_mono", [False, True])
def test_coset_sharded_lde(bj, from_mono):
    """set_coset_shard(rank, world, 8): bj_lde writes the cosets j = rank (mod world) of the unsharded LDE, in order."""
    log_n, cols = 12, 3
    a = field_input(1200 + from_mono, (cols, 1 << log_n))
    want = O.lde(a, 3, from_monomials=from_mono)
    with context(bj) as c:
        for world in (2, 4, 8):
            for rank in range(world):
                c.set_coset_shard(rank, world, 8)
                out = c.transform_raw_storages_to_lde(bj.to_device(a), 8, from_monomials=from_mono)
                check(bj.to_numpy(out), want[:, rank::world])


def test_coset_sharded_lde_wider_domain(bj):
    """A shard declared for an LDE factor of 2 over 2 ranks, asked for 8 cosets (the quotient's wider domain): each rank
    gets its 4 cosets j = rank (mod 2), in order."""
    log_n, cols = 12, 2
    a = field_input(1300, (cols, 1 << log_n))
    want = O.lde(a, 3)
    with context(bj) as c:
        for rank in range(2):
            c.set_coset_shard(rank, 2, 2)
            out = c.transform_raw_storages_to_lde(bj.to_device(a), 8)
            assert out.shape == (cols, 4, 1 << log_n)
            check(bj.to_numpy(out), want[:, rank::2])
