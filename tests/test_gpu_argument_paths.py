"""GPU tests of the stage-2, lookup, quotient, opening, DEEP, FRI-fold and batch-inverse kernels at the sizes and
geometries where their less common code paths switch on:
  - stage 2: the pass-2 scan over more than 256 scan blocks (n > 2^19 rows), and the copy-permutation quotient at
    Q = 1, Q < L, Q = L = 8, one chunk and 155 columns;
  - the lookup argument with up to 32 sub-arguments and tuples of 8 columns (gamma^5..gamma^7);
  - the barycentric dot product's grid-stride loop (rows > 4 * SMs * 256) and a partial last column tile;
  - the DEEP accumulator's overflow word (hundreds of columns at full magnitude) and its column tail at 2^21 / 2^23 rows;
  - FRI folds and batch inversion at prover sizes.

Every output is compared over the whole vector with the C oracle (oracle/oracle.c, pinned to the Python-int oracles by
tests/test_oracle_arguments_cpu.py) and checked to be canonical.  Inputs carry non-canonical representatives wherever the
kernel takes lazy input: p is added to a seeded subset of the cells below 2^32 - 1, which keeps the field element, so a
satisfying witness stays satisfying."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import stage2 as S

pytestmark = pytest.mark.gpu

P = O.P
P_I64 = P - 2**64          # p as the int64 that torch stores: adding it to v < 2^32 - 1 gives the bits of v + p
INVALID_ARG = -1


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


@pytest.fixture(scope="module")
def ctx(bj):
    c = bj.Context.on_current_stream(0)
    yield c
    c.synchronize()
    c.close()


def rng(seed):
    return np.random.default_rng(seed)


def e2(r):
    return tuple(int(x) for x in O.random_field(r, 2))


def wide(r, shape, frac=0.05):
    """uniform 64-bit words with a planted share of non-canonical values in [p, 2^64) (for pointwise kernels)"""
    a = r.integers(0, 2**64, size=shape, dtype=np.uint64)
    flat = a.reshape(-1)
    k = max(1, int(frac * flat.size))
    flat[r.integers(0, flat.size, size=k)] = r.integers(P, 2**64, size=k, dtype=np.uint64)
    return a


def lazy_np(r, a, frac=0.25):
    """a (canonical) with p added to a seeded subset of its cells below 2^32 - 1: same field elements"""
    a = np.array(a, dtype=np.uint64)
    flat = a.reshape(-1)
    small = np.flatnonzero(flat < np.uint64(2**32 - 1))
    flat[small[r.random(small.size) < frac]] += np.uint64(P)
    return a


def lazy_dev(t, seed, frac=0.25):
    """lazy_np for an int64 CUDA tensor, in place"""
    import torch
    gen = torch.Generator(device=t.device)
    gen.manual_seed(seed)
    mask = (t >= 0) & (t < 2**32 - 1) & (torch.rand(t.shape, generator=gen, device=t.device) < frac)
    assert mask.any()
    t.copy_(torch.where(mask, t + P_I64, t))
    return t


def lazy_sigmas(t, seed):
    """lazy_dev for sigma columns: sigma = k_j' * omega^i' is below 2^32 - 1 only where it names a row-0 cell (k_j' is a
    small integer), so every such cell gets its non-canonical representative"""
    return lazy_dev(t, seed + 1, frac=1.0)


def assert_canonical(*arrays):
    for a in arrays:
        assert (np.asarray(a) < np.uint64(P)).all(), "non-canonical output"


def assert_equal(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert_canonical(got)
    if not np.array_equal(got, want):
        bad = np.flatnonzero(got.reshape(-1) != want.reshape(-1))
        raise AssertionError("%s: %d of %d values differ, first at %d" % (what, bad.size, want.size, bad[0]))


def field_sum(a):
    """sum of a uint64 vector mod p (exact: 32-bit halves summed in uint64)"""
    a = np.asarray(a, dtype=np.uint64)
    lo = int((a & np.uint64(0xFFFFFFFF)).sum(dtype=np.uint64))
    hi = int((a >> np.uint64(32)).sum(dtype=np.uint64))
    assert a.size < 2**31
    return ((hi << 32) + lo) % P


# ------------------------------------------------------------------------------------------------ stage 2 -----
def identity_sigmas(n_cols, log_n):
    """k_j * omega^i (natural order) from the oracle's NTT of the polynomials k_j * X"""
    n = 1 << log_n
    ks = S.non_residues_for_copy_permutation(n, n_cols)
    mono = np.zeros((n_cols, n), np.uint64)
    mono[:, 1] = ks
    return O.bitreverse(O.ntt_n2b(mono))


def paired_copy_permutation(bj, n_cols, log_n, seed):
    """columns (2a, 2a + 1) tied by a random row permutation pi: cell (2a + 1, i) holds the value of (2a, pi(i)) and the two
    cells form one cycle, so every ratio is non-trivial and the grand product is one.  A last odd column is its own cycle."""
    n = 1 << log_n
    r = rng(seed)
    ident = identity_sigmas(n_cols, log_n)
    vals = r.integers(0, 2**36, size=(n_cols, n), dtype=np.uint64)
    sig = ident.copy()
    for a in range(0, n_cols - 1, 2):
        pi = r.permutation(n)
        vals[a + 1] = vals[a][pi]
        sig[a + 1] = ident[a][pi]
        sig[a][pi] = ident[a + 1]
    d_v, d_s = bj.to_device(vals), bj.to_device(sig)
    return lazy_dev(d_v, seed), lazy_sigmas(d_s, seed)


def check_stage2(bj, ctx, variables, sigmas, chunk, seed):
    """compute_partial_products_in_extension on [V, n] device columns against orc_cp_stage2, every row"""
    V, n = variables.shape
    r = rng(seed)
    beta, gamma = e2(r), e2(r)
    z0, z1, partials = ctx.compute_partial_products_in_extension([variables[c] for c in range(V)], [sigmas[c] for c in range(V)],
                                                                 beta, gamma, chunk)
    hv, hs = bj.to_numpy(variables), bj.to_numpy(sigmas)
    assert (hv >= np.uint64(P)).any(), "the witness carries no non-canonical cell"
    assert (hs >= np.uint64(P)).any(), "sigma carries no non-canonical cell"
    w0, w1, wp, grand = O.cp_stage2(list(hv), list(hs), S.non_residues_for_copy_permutation(n, V), beta, gamma, chunk)
    del hv, hs
    assert grand == (1, 0)
    assert len(partials) == len(wp) == (V + chunk - 1) // chunk - 1
    assert_equal(bj.to_numpy(z0), w0, "z.c0")
    assert_equal(bj.to_numpy(z1), w1, "z.c1")
    for c, (p0, p1) in enumerate(partials):
        assert_equal(bj.to_numpy(p0), wp[c, 0], "partial %d c0" % c)
        assert_equal(bj.to_numpy(p1), wp[c, 1], "partial %d c1" % c)


@pytest.mark.parametrize("log_n", [11, 12, 19, 20, 22])
def test_stage2_scan_block_boundaries(bj, ctx, log_n):
    """2^11 rows fill one scan block, 2^12 two; 2^19 rows are exactly 256 blocks (one pass of the scan of block products),
    2^20 rows 512 (the carry crosses one 256-block chunk), 2^22 rows 2048 (eight passes).  The synthetic circuits below
    tie cells of the same row only, so their row products are all one and z is constant: these cycles cross rows, so
    every block product, and so the carry, is a non-trivial value."""
    variables, sigmas = paired_copy_permutation(bj, 5, log_n, seed=log_n)
    check_stage2(bj, ctx, variables, sigmas, 2, seed=log_n)


@pytest.fixture(scope="module")
def bench22(bj, ctx):
    """the SHA-bench-shaped circuit at 2^22 rows, 60 columns (2048 scan blocks: the pass-2 loop runs 8 times).  Its copy
    cycles stay inside a row, so z is one on every row; the ratios and partial products are not."""
    from era_boojum_b200 import synthetic
    variables, sigmas, constants, gates, Q = synthetic.generate(ctx, 22, 60)
    return lazy_dev(variables, 22), lazy_sigmas(sigmas, 22), constants, Q


def test_stage2_sha_bench_2p22(bj, ctx, bench22):
    variables, sigmas, _, Q = bench22
    check_stage2(bj, ctx, variables, sigmas, Q, seed=2201)


def test_stage2_rejects_a_broken_copy_in_the_last_scan_block(bj, ctx, bench22):
    """One FMA row in the last scan block gets a different value in column 6, which is tied to column 3 on FMA rows."""
    variables, sigmas, constants, Q = bench22
    n = variables.shape[1]
    fma_rows = ((constants[0] == 1) & (constants[1] == 0)).nonzero().flatten()
    row = int(fma_rows[-1])
    assert row >= n - 2048
    broken = variables.clone()
    broken[6, row] += 1
    with pytest.raises(bj.BoojumError) as e:
        ctx.compute_partial_products_in_extension([broken[c] for c in range(60)], [sigmas[c] for c in range(60)], e2(rng(1)), e2(rng(2)), Q)
    assert e.value.status == INVALID_ARG and "grand product" in str(e.value)


def test_stage2_production_shape_2p20(bj, ctx):
    """155 columns, chunk 8: 20 chunks, 19 partial products"""
    from era_boojum_b200 import synthetic
    c = synthetic.generate_production_shaped(ctx, 20)
    variables = lazy_dev(c["variables"], 20)
    assert variables.shape[0] == 155
    check_stage2(bj, ctx, variables, lazy_sigmas(c["sigmas"], 20), c["quotient_degree"], seed=2001)


# ------------------------------------------------------------------------------ copy-permutation quotient -----
@pytest.mark.parametrize("n_cols,chunk,log_n,log_lde,log_q", [
    (17, 8, 20, 3, 3),     # production rows, Q = L = 8, last chunk partial
    (155, 8, 12, 3, 3),    # production column count over 8 cosets
    (6, 8, 12, 2, 1),      # one chunk
    (9, 4, 14, 1, 0),      # Q = 1
    (10, 3, 16, 3, 2),     # Q < L
], ids=["2p20-Q8-L8", "155cols", "one-chunk", "Q1", "Q-below-L"])
def test_quotient_copy_permutation_and_division(bj, ctx, n_cols, chunk, log_n, log_lde, log_q):
    """The relation is pointwise, so random LDE columns (non-canonical values included) are enough."""
    r = rng(1000 * n_cols + 10 * log_n + log_q)
    n_chunks = (n_cols + chunk - 1) // chunk
    full, npts = 1 << (log_n + log_lde), 1 << (log_n + log_q)
    v, s = wide(r, (n_cols, full)), wide(r, (n_cols, full))
    z = wide(r, (2, full))
    part = wide(r, (max(n_chunks - 1, 1), 2, full))
    beta, gamma = e2(r), e2(r)
    alphas = [e2(r) for _ in range(n_chunks + 1)]
    init = wide(r, (2, npts))
    dv, ds, dz, dp, dq = (bj.to_device(x) for x in (v, s, z, part, init))
    ctx.quotient_copy_permutation([dv[c] for c in range(n_cols)], [ds[c] for c in range(n_cols)], (dz[0], dz[1]),
                                  [(dp[c, 0], dp[c, 1]) for c in range(n_chunks - 1)], beta, gamma, alphas, log_n, log_lde, log_q,
                                  chunk, dq[0], dq[1])
    got = bj.to_numpy(dq)
    del dv, ds, dz, dp
    ks = S.non_residues_for_copy_permutation(1 << log_n, n_cols)
    w0, w1 = O.cp_quotient(list(v), list(s), ks, (z[0], z[1]), [(part[c, 0], part[c, 1]) for c in range(n_chunks - 1)], beta, gamma,
                           alphas, log_n, log_lde, log_q, chunk, init[0], init[1])
    del v, s, z, part
    assert_equal(got[0], w0, "q.c0")
    assert_equal(got[1], w1, "q.c1")
    # the division takes lazy input as well
    lz = np.stack([lazy_np(r, w0, 0.5), lazy_np(r, w1, 0.5)])
    lz[:, :64] = np.uint64(7) + np.uint64(P)
    dq = bj.to_device(lz)
    ctx.divide_by_vanishing(dq[0], dq[1], log_n, log_q)
    got = bj.to_numpy(dq)
    d0, d1 = O.divide_by_vanishing(lz[0], lz[1], log_n, log_q)
    assert_equal(got[0], d0, "divided c0")
    assert_equal(got[1], d1, "divided c1")


# ----------------------------------------------------------------------------------------------- lookup -----
LOOKUP_GEOMETRIES = [(8, 3, True), (8, 4, True), (32, 7, True), (32, 8, False), (1, 1, False)]


@pytest.mark.parametrize("n_sub,width,with_id", LOOKUP_GEOMETRIES, ids=["production", "bench", "32x7+id", "32x8", "1x1"])
def test_lookup_polys_and_quotient_2p20(bj, ctx, n_sub, width, with_id):
    """A_i / B and the quotient terms at 2^20 points on random columns (the formulas are pointwise), all inputs lazy."""
    log_n = 20
    n = 1 << log_n
    r = rng(100 * n_sub + 10 * width + with_id)
    n_tab = width + int(with_id)
    cols = wide(r, (n_sub * width, n))
    tid = wide(r, n) if with_id else None
    tabs, mult = wide(r, (n_tab, n)), wide(r, n)
    beta, gamma = e2(r), e2(r)
    d_cols, d_tabs, d_mult = bj.to_device(cols), bj.to_device(tabs), bj.to_device(mult)
    d_tid = bj.to_device(tid) if with_id else None
    A, B = ctx.compute_lookup_poly_pairs_specialized([d_cols[i] for i in range(n_sub * width)], width, d_tid,
                                                     [d_tabs[i] for i in range(n_tab)], d_mult, beta, gamma)
    want = O.lookup_polys(list(cols), width, tid, list(tabs), mult, beta, gamma)
    for i in range(n_sub):
        assert_equal(bj.to_numpy(A[i][0]), want[i, 0], "A_%d c0" % i)
        assert_equal(bj.to_numpy(A[i][1]), want[i, 1], "A_%d c1" % i)
    assert_equal(bj.to_numpy(B[0]), want[n_sub, 0], "B c0")
    assert_equal(bj.to_numpy(B[1]), want[n_sub, 1], "B c1")
    del A, B, want
    # quotient terms, on the same columns taken as LDE values, with random A / B
    a = wide(r, (n_sub, 2, n))
    b = wide(r, (2, n))
    alphas = [e2(r) for _ in range(n_sub + 1)]
    init = wide(r, (2, n))
    da, db, dq = bj.to_device(a), bj.to_device(b), bj.to_device(init)
    ctx.quotient_lookup_specialized([d_cols[i] for i in range(n_sub * width)], width, d_tid, [d_tabs[i] for i in range(n_tab)], d_mult,
                                    [(da[i, 0], da[i, 1]) for i in range(n_sub)], (db[0], db[1]), beta, gamma, alphas, dq[0], dq[1])
    got = bj.to_numpy(dq)
    w0, w1 = O.lookup_quotient(list(cols), width, tid, list(tabs), mult, [(a[i, 0], a[i, 1]) for i in range(n_sub)], (b[0], b[1]),
                               beta, gamma, alphas, init[0], init[1])
    assert_equal(got[0], w0, "lookup quotient c0")
    assert_equal(got[1], w1, "lookup quotient c1")


@pytest.mark.parametrize("n_sub,width,with_id", [(33, 1, False), (33, 3, True), (1, 8, True), (2, 9, False)])
def test_lookup_geometry_limits_are_refused(bj, ctx, n_sub, width, with_id):
    """more than 32 sub-arguments, or tuples wider than 8 columns with the table id, return BJ_ERR_INVALID_ARG"""
    import torch
    n = 1 << 6
    col = torch.ones(n, dtype=torch.int64, device="cuda:0")
    n_tab = width + int(with_id)
    tid = col if with_id else None
    with pytest.raises(bj.BoojumError) as e:
        ctx.compute_lookup_poly_pairs_specialized([col] * (n_sub * width), width, tid, [col] * n_tab, col, (1, 2), (3, 4))
    assert e.value.status == INVALID_ARG
    q = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    with pytest.raises(bj.BoojumError) as e:
        ctx.quotient_lookup_specialized([col] * (n_sub * width), width, tid, [col] * n_tab, col, [(col, col)] * n_sub, (col, col),
                                        (1, 2), (3, 4), [(5, 6)] * (n_sub + 1), q, q)
    assert e.value.status == INVALID_ARG
    assert not q.any()


def test_lookup_log_derivative_identity_on_the_2p22_bench_circuit(bj, ctx):
    """sum over rows of sum_i A_i equals sum over rows of B when every tuple is a table row and m counts them"""
    from era_boojum_b200 import synthetic
    variables, sigmas, constants, gates, Q, lk = synthetic.generate(ctx, 22, 60, seed=5, lookup=True)
    del sigmas
    width, n_sub, off = lk["width"], lk["num_repetitions"], lk["variables_offset"]
    lk_cols = lazy_dev(variables[off:off + n_sub * width].contiguous(), 5)
    del variables
    tables = lk["tables"]
    r = rng(22)
    A, B = ctx.compute_lookup_poly_pairs_specialized([lk_cols[i] for i in range(n_sub * width)], width,
                                                     constants[lk["table_id_column"]].contiguous(),
                                                     [tables[j] for j in range(width + 1)], lk["multiplicities"], e2(r), e2(r))
    lhs = [0, 0]
    for a in A:
        for k in (0, 1):
            h = bj.to_numpy(a[k])
            assert_canonical(h)
            lhs[k] = (lhs[k] + field_sum(h)) % P
    rhs = [field_sum(bj.to_numpy(B[k])) for k in (0, 1)]
    assert lhs == rhs
    assert lhs != [0, 0]


# -------------------------------------------------------------------------------------------- barycentric -----
def coset0_and_monomials(r, n_cols, log_n):
    """values of random polynomials on coset 0 of the LDE (7 * w_n^{bitrev(i)}, bit-reversed, some lazy) and their
    monomials from the oracle's iNTT"""
    n = 1 << log_n
    vals, mono = np.empty((n_cols, n), np.uint64), np.empty((n_cols, n), np.uint64)
    for c0 in range(0, n_cols, 16):          # in groups of columns, to keep host memory low
        k = min(16, n_cols - c0)
        vals[c0:c0 + k] = lazy_np(r, O.random_field(r, (k, n)) >> r.integers(0, 40, size=(k, n), dtype=np.uint64))
        mono[c0:c0 + k] = O.intt_n2n(O.bitreverse(vals[c0:c0 + k]), coset=7)
    return vals, mono


def check_barycentric(bj, ctx, vals, mono, log_n, r):
    d = bj.to_device(vals)
    cols = [d[c] for c in range(vals.shape[0])]
    for at in (e2(r), (0, 0), (int(O.random_field(r, 1)[0]), 0)):
        got = np.array(ctx.barycentric_evaluate(cols, log_n, at), dtype=np.uint64)
        assert_equal(got, O.horner_ext(mono, at), "f(%s)" % (at,))


@pytest.mark.parametrize("log_n", [17, 18, 20, 21])
def test_barycentric_grid_stride_rows(bj, ctx, log_n):
    """from 2^18 rows on, a thread of the dot product accumulates more than one row (grid capped at 4 blocks per SM)"""
    r = rng(log_n)
    vals, mono = coset0_and_monomials(r, 3, log_n)
    check_barycentric(bj, ctx, vals, mono, log_n, r)


def test_barycentric_155_columns_2p20(bj, ctx):
    """155 columns: grid.y = 20 column tiles of 8, the last one holds 3"""
    r = rng(155)
    vals, mono = coset0_and_monomials(r, 155, 20)
    check_barycentric(bj, ctx, vals, mono, 20, r)


# --------------------------------------------------------------------------------------------------- DEEP -----
def check_deep(bj, ctx, srcs, vals, chs, at, acc):
    """srcs: list of (c0, c1 or None) host columns"""
    d_srcs = [(bj.to_device(s0), bj.to_device(s1) if s1 is not None else None) for s0, s1 in srcs]
    g0, g1 = ctx.quotening_operation_in_extension(bj.to_device(acc[0]), bj.to_device(acc[1]), d_srcs, vals, at, chs)
    got0, got1 = bj.to_numpy(g0), bj.to_numpy(g1)
    del d_srcs, g0, g1
    w0, w1 = O.deep_group(acc[0], acc[1], srcs, vals, chs, at)
    assert_equal(got0, w0, "DEEP c0")
    assert_equal(got1, w1, "DEEP c1")


@pytest.mark.parametrize("extra_base", [0, 1, 2, 3])
@pytest.mark.parametrize("extreme", [False, True], ids=["random", "full-magnitude"])
def test_deep_hundreds_of_columns(bj, ctx, extra_base, extreme):
    """The fixture's 374 DEEP sources (327 base-field, 47 extension: 421 flattened columns), plus 1-3 more base columns so
    that the flattened count is 1, 2, 3 and 0 (mod 4).  full-magnitude: every source in [p, 2^64) and every challenge
    p - 1, so each product is close to 2^128 and the accumulator's overflow word passes 255."""
    log_rows = 16
    rows = 1 << log_rows
    r = rng(374 + extra_base + 10 * extreme)
    n_base, n_ext = 327 + extra_base, 47
    n = n_base + n_ext
    col = (lambda: r.integers(P, 2**64, size=rows, dtype=np.uint64)) if extreme else (lambda: wide(r, rows))
    srcs = [(col(), None) for _ in range(n_base)] + [(col(), col()) for _ in range(n_ext)]
    vals = [e2(r) for _ in range(n)]
    chs = [(P - 1, P - 1)] * n if extreme else [e2(r) for _ in range(n)]
    check_deep(bj, ctx, srcs, vals, chs, e2(r), wide(r, (2, rows)))


@pytest.mark.parametrize("log_rows", [21, 23])
def test_deep_large_domain(bj, ctx, log_rows):
    """10 sources (6 base, 4 extension: 14 flattened columns, a tail of 2 after the groups of 4) at 2^21 and 2^23 points"""
    rows = 1 << log_rows
    r = rng(log_rows)
    srcs = [(wide(r, rows), None) for _ in range(6)] + [(wide(r, rows), wide(r, rows)) for _ in range(4)]
    vals = [e2(r) for _ in range(10)]
    chs = [e2(r) for _ in range(9)] + [(P - 1, P - 1)]
    check_deep(bj, ctx, srcs, vals, chs, e2(r), wide(r, (2, rows)))


# ----------------------------------------------------------------------------------------------- FRI fold -----
def oracle_fold(c0, c1, k, alpha, kappa, roots):
    w0, w1, a = c0, c1, tuple(alpha)
    for _ in range(k):
        w0, w1 = O.fri_fold(w0, w1, a, roots[: len(w0) // 2], kappa)
        a, kappa = O.ext_mul(a, a), O.mul(kappa, kappa)
    return w0, w1, kappa


@pytest.mark.parametrize("log_m", [21, 23])
def test_fri_fold_by_8_at_prover_sizes(bj, ctx, log_m):
    r = rng(log_m)
    c0, c1 = wide(r, 1 << log_m), wide(r, 1 << log_m)
    alpha = list(e2(r))
    o0, o1, kappa = ctx.fri_fold(bj.to_device(c0), bj.to_device(c1), 3, alpha, O.inv(7))
    w0, w1, wk = oracle_fold(c0, c1, 3, alpha, O.inv(7), O.twiddles(log_m, inverse=True))
    assert_equal(bj.to_numpy(o0), w0, "fold c0")
    assert_equal(bj.to_numpy(o1), w1, "fold c1")
    assert kappa == wk


def test_fri_fold_chain_3_2_1(bj, ctx):
    """one codeword folded 3, 2 and 1 times in a row, as do_fri does: every level uses a prefix of the full domain's roots
    and the coset inverse the previous step returned"""
    log_m = 23
    r = rng(321)
    c0, c1 = wide(r, 1 << log_m), wide(r, 1 << log_m)
    roots = O.twiddles(log_m, inverse=True)
    d0, d1, kappa = bj.to_device(c0), bj.to_device(c1), O.inv(7)
    w0, w1, wk = c0, c1, O.inv(7)
    for k in (3, 2, 1):
        alpha = list(e2(r))
        d0, d1, kappa = ctx.fri_fold(d0, d1, k, alpha, kappa)
        w0, w1, wk = oracle_fold(w0, w1, k, alpha, wk, roots)
        assert_equal(bj.to_numpy(d0), w0, "fold-by-%d c0" % (1 << k))
        assert_equal(bj.to_numpy(d1), w1, "fold-by-%d c1" % (1 << k))
        assert kappa == wk


# ------------------------------------------------------------------------------------------ batch inverse -----
def test_batch_inverse_ragged_with_zeros_and_lazy_values(bj, ctx):
    n = (1 << 22) + 3
    r = rng(223)
    a = O.random_field(r, n)
    small = r.random(n) < 0.05
    a[small] = r.integers(1, 2**32 - 1, size=int(small.sum()), dtype=np.uint64)
    a = lazy_np(r, a, 0.5)
    zeros = r.choice(n, 1000, replace=False)
    a[zeros[:500]] = 0
    a[zeros[500:]] = P                       # a non-canonical zero
    a[-1] = 0
    got = bj.to_numpy(ctx.batch_inverse_inplace(bj.to_device(a)))
    nz = (a % np.uint64(P)) != 0
    want = np.zeros(n, np.uint64)
    want[nz] = O.batch_inverse(a[nz])
    assert_equal(got, want, "batch inverse")


def test_batch_inverse_ext_ragged_with_zeros_and_lazy_values(bj, ctx):
    n = (1 << 22) + 3
    r = rng(224)
    c = O.random_field(r, (2, n))
    small = r.random((2, n)) < 0.05
    c[small] = r.integers(1, 2**32 - 1, size=int(small.sum()), dtype=np.uint64)
    c = lazy_np(r, c, 0.5)
    cells = r.choice(n, 1600, replace=False).reshape(8, 200)
    c[:, cells[0]] = 0
    c[:, cells[1]] = P
    c[0, cells[2]], c[1, cells[2]] = 0, P
    c[0, cells[3]], c[1, cells[3]] = P, 0
    c[0, cells[4]] = 0                        # one zero component: not zero
    c[1, cells[5]] = P
    c[:, -1] = 0
    g0, g1 = ctx.batch_inverse_inplace_in_extension(bj.to_device(c[0]), bj.to_device(c[1]))
    nz = ((c[0] % np.uint64(P)) != 0) | ((c[1] % np.uint64(P)) != 0)
    w0, w1 = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    w0[nz], w1[nz] = O.batch_inverse_ext(c[0][nz], c[1][nz])
    assert_equal(bj.to_numpy(g0), w0, "batch inverse ext c0")
    assert_equal(bj.to_numpy(g1), w1, "batch inverse ext c1")
