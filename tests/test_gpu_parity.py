"""GPU parity tests: the CUDA path, called through the C-ABI (era_boojum_b200 -> libboojum_b200.so), against the CPU
oracle on the same seeded inputs, against the reference's golden fixture, and - at BASELINE.json sizes - through
size-independent properties.  Bit-exact: all values are integers mod p compared after canonicalisation."""
import os
import numpy as np
import pytest

from oracle import oracle as O
from oracle import replay

pytestmark = pytest.mark.gpu

P = O.P


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


# ------------------------------------------------------------------------------------------- NTT -------
def test_twiddles_match_reference_table(bj, ctx):
    for log_n in (1, 2, 5, 12, 16):
        for inv in (False, True):
            got = bj.to_numpy(ctx.precompute_twiddles_for_fft(1 << log_n, inv))
            assert np.array_equal(got[: max(1, (1 << log_n) // 2)], O.twiddles(log_n, inv))


@pytest.mark.parametrize("log_n", list(range(0, 22)))
@pytest.mark.parametrize("coset", [1, 7])
def test_ntt_forward_matches_oracle(bj, ctx, log_n, coset):
    n_cols = 3 if log_n <= 16 else 2
    a = O.random_field(rng(log_n * 2 + coset), (n_cols, 1 << log_n))
    d = bj.to_device(a)
    ctx.fft_natural_to_bitreversed(d, coset)
    assert np.array_equal(bj.to_numpy(d), O.ntt_n2b(a, coset))


@pytest.mark.parametrize("log_n", list(range(0, 22)))
@pytest.mark.parametrize("coset", [1, 7])
def test_ntt_inverse_matches_oracle(bj, ctx, log_n, coset):
    n_cols = 3 if log_n <= 16 else 2
    a = O.random_field(rng(1000 + log_n * 2 + coset), (n_cols, 1 << log_n))
    d = bj.to_device(a)
    ctx.ifft_natural_to_natural(d, coset)
    assert np.array_equal(bj.to_numpy(d), O.intt_n2n(a, coset))


def test_ntt_config1_2pow16_forward_inverse(bj, ctx):
    """BASELINE config 1: 2^16-point forward + inverse, cosets 1 and 7, adversarial inputs incl. non-canonical
    values in [p, 2^64) (reference: src/field/goldilocks/generic_impl.rs:449-455) and 0/1 vectors (fft/mod.rs:1432)."""
    n = 1 << 16
    r = rng(16)
    cases = [
        O.random_field(r, n),
        np.zeros(n, np.uint64),
        np.full(n, P - 1, np.uint64),
        r.integers(P, 2**64, size=n, dtype=np.uint64),       # all non-canonical
        np.full(n, 2**64 - 1, np.uint64),
        (np.arange(n) % 2).astype(np.uint64),
        np.concatenate([np.ones(1, np.uint64), np.zeros(n - 1, np.uint64)]),
    ]
    a = np.stack(cases)
    for coset in (1, 7):
        d = bj.to_device(a)
        ctx.fft_natural_to_bitreversed(d, coset)
        fwd = bj.to_numpy(d)
        assert np.array_equal(fwd, O.ntt_n2b(a, coset))
        assert (fwd < np.uint64(P)).all()
        d = bj.to_device(a)
        ctx.ifft_natural_to_natural(d, coset)
        assert np.array_equal(bj.to_numpy(d), O.intt_n2n(a, coset))
        # round trip: iNTT(bitrev(NTT(a))) == a mod p
        d = bj.to_device(a)
        ctx.fft_natural_to_bitreversed(d, coset)
        ctx.bitreverse_enumeration_inplace(d)
        ctx.ifft_natural_to_natural(d, coset)
        assert np.array_equal(bj.to_numpy(d), a % np.uint64(P))


@pytest.mark.parametrize("log_n", [14, 20, 22, 24])
def test_ntt_bulk_copy_staged_pass_matches_oracle(bj, log_n, monkeypatch):
    """BJ_NTT_BULK=1: the contiguous pass moved by cp.async.bulk + mbarrier (the TMA experiment, ntt_v2.cuh) gives the same
    transform bit for bit (forward with and without coset, inverse, LDE)."""
    monkeypatch.setenv("BJ_NTT_BULK", "1")
    c = bj.Context.on_current_stream(0)
    try:
        a = O.random_field(rng(900 + log_n), (2, 1 << log_n))
        for coset in (1, 7):
            d = bj.to_device(a)
            c.fft_natural_to_bitreversed(d, coset)
            assert np.array_equal(bj.to_numpy(d), O.ntt_n2b(a, coset))
        d = bj.to_device(a)
        c.ifft_natural_to_natural(d, 7)
        assert np.array_equal(bj.to_numpy(d), O.intt_n2n(a, 7))
        if log_n <= 20:
            assert np.array_equal(bj.to_numpy(c.transform_raw_storages_to_lde(bj.to_device(a), 4)), O.lde(a, 2))
    finally:
        c.synchronize()
        c.close()


def test_ntt_strided_batch(bj, ctx):
    """columns separated by a stride larger than n (col_stride argument of the C-ABI)."""
    import ctypes
    import torch
    from era_boojum_b200 import native
    n, cols, stride = 1 << 13, 4, (1 << 13) + 64
    a = O.random_field(rng(5), (cols, n))
    buf = np.zeros(cols * stride, np.uint64)
    for c in range(cols):
        buf[c * stride: c * stride + n] = a[c]
    buf[n:stride] = 12345  # padding must stay untouched
    d = bj.to_device(buf)
    st = native.lib.bj_ntt_natural_to_bitreversed(ctx._h, ctypes.c_void_p(d.data_ptr()), 13, cols, stride, 7)
    assert st == 0
    out = bj.to_numpy(d)
    want = O.ntt_n2b(a, 7)
    for c in range(cols):
        assert np.array_equal(out[c * stride: c * stride + n], want[c])
    assert (out[n:stride] == 12345).all()
    torch.cuda.synchronize()


def _add_mod(x, y):
    """(x + y) mod p element-wise for canonical uint64 arrays (exact; numpy wraps the 64-bit sum)."""
    s = x + y
    return np.where((s < x) | (s >= np.uint64(P)), s - np.uint64(P), s)


@pytest.mark.parametrize("log_n", [21, 22, 23, 24, 25, 26])
def test_ntt_full_size_vs_oracle_and_properties(bj, ctx, log_n):
    """BASELINE config 2 sizes: one column compared with the oracle directly, plus linearity and round trip.  2^25 and
    2^26 are the first three-pass forward plans."""
    n = 1 << log_n
    r = rng(log_n)
    a, b = O.random_field(r, n), O.random_field(r, n)
    d = bj.to_device(np.stack([a, b]))
    ctx.fft_natural_to_bitreversed(d, 7)
    fa, fb = bj.to_numpy(d)
    assert np.array_equal(fa, O.ntt_n2b(a, 7))
    # linearity: NTT(a + 3b) == NTT(a) + 3 NTT(b)
    lin = _add_mod(a, _add_mod(b, _add_mod(b, b)))
    d2 = bj.to_device(lin)
    ctx.fft_natural_to_bitreversed(d2, 7)
    want = _add_mod(fa, _add_mod(fb, _add_mod(fb, fb)))
    assert np.array_equal(bj.to_numpy(d2), want)
    # round trip
    ctx.bitreverse_enumeration_inplace(d)
    ctx.ifft_natural_to_natural(d, 7)
    back = bj.to_numpy(d)
    assert np.array_equal(back[0], a) and np.array_equal(back[1], b)
    # inverse against the oracle at full size too
    d3 = bj.to_device(a)
    ctx.ifft_natural_to_natural(d3, 7)
    assert np.array_equal(bj.to_numpy(d3), O.intt_n2n(a, 7))


# ------------------------------------------------------------------------------------------- LDE -------
@pytest.mark.parametrize("log_n,log_l,cols", [(4, 1, 2), (10, 3, 5), (13, 2, 3), (16, 3, 3)])
def test_lde_matches_oracle(bj, ctx, log_n, log_l, cols):
    a = O.random_field(rng(log_n + log_l), (cols, 1 << log_n))
    d = bj.to_device(a)
    out = ctx.transform_raw_storages_to_lde(d, 1 << log_l)
    assert np.array_equal(bj.to_numpy(out), O.lde(a, log_l))
    assert np.array_equal(bj.to_numpy(d), a)  # input untouched
    mono = O.intt_n2n(a)
    out2 = ctx.transform_raw_storages_to_lde(bj.to_device(mono), 1 << log_l, from_monomials=True)
    assert np.array_equal(bj.to_numpy(out2), O.lde(a, log_l))


def test_lde_large_first_coset_subset(bj, ctx):
    """n = 2^20, L = 8: the first 2 cosets equal the L = 2 LDE (subset_for_degree, polynomial/lde.rs:298-308) and one
    coset is checked against the oracle."""
    log_n = 20
    a = O.random_field(rng(77), (2, 1 << log_n))
    d = bj.to_device(a)
    out8 = bj.to_numpy(ctx.transform_raw_storages_to_lde(d, 8))
    out2 = bj.to_numpy(ctx.transform_raw_storages_to_lde(d, 2))
    assert np.array_equal(out8[:, :2, :], out2)
    want = O.lde(a[:1], 3)
    assert np.array_equal(out8[0], want[0])


def test_lde_prover_shape_2pow22_factor8_vs_oracle(bj, ctx):
    """The prover's LDE shape (BASELINE configs[3]/[4]): n = 2^22, L = 8; 8 columns go through bj_lde together (so the
    batched/fused code path is the one that runs) and one column is compared with the oracle on all 8 cosets."""
    log_n = 22
    a = O.random_field(rng(2208), (8, 1 << log_n))
    d = bj.to_device(a)
    out = bj.to_numpy(ctx.transform_raw_storages_to_lde(d, 8))
    want = O.lde(a[5:6], 3)
    assert np.array_equal(out[5], want[0])
    # the other columns: cosets are NTTs of the same monomials -> check coset 0 of each column against a forward NTT
    mono = O.intt_n2n(a[:2])
    assert np.array_equal(out[0, 0], O.ntt_n2b(mono[0], 7))
    assert np.array_equal(out[1, 0], O.ntt_n2b(mono[1], 7))


# ------------------------------------------------------------------------------------ Poseidon2 / Merkle -----
def test_poseidon2_permutation_matches_oracle(bj, ctx):
    r = rng(8)
    st = r.integers(0, 2**64, size=(300, 12), dtype=np.uint64)
    st[::7, ::3] = r.integers(P, 2**64, size=st[::7, ::3].shape, dtype=np.uint64)  # non-canonical words in the checked rows
    d = bj.to_device(st)
    ctx.poseidon2_permute(d)
    got = bj.to_numpy(d)
    for i in range(0, 300, 7):
        assert np.array_equal(got[i], O.poseidon2_permutation(st[i]))


@pytest.mark.parametrize("row_len", [1, 4, 7, 8, 9, 16, 58, 93, 156])
def test_poseidon2_leaf_hash_rows(bj, ctx, row_len):
    rows = O.random_field(rng(row_len), (33, row_len))
    got = bj.to_numpy(ctx.poseidon2_hash_rows(bj.to_device(rows)))
    for i in range(33):
        assert np.array_equal(got[i], O.poseidon2_hash_leaf(rows[i]))


@pytest.mark.parametrize("n_cols,log_leaves,cap", [(1, 4, 1), (8, 6, 4), (11, 8, 16), (93, 12, 16), (100, 10, 1024)])
def test_merkle_tree_matches_oracle(bj, ctx, n_cols, log_leaves, cap):
    n = 1 << log_leaves
    cols = [O.random_field(rng(100 * n_cols + c), n) for c in range(n_cols)]
    tree = ctx.merkle_tree_construct([bj.to_device(c) for c in cols], cap)
    lh, levels, capd = O.merkle_tree(cols, cap)
    assert np.array_equal(bj.to_numpy(tree.leaf_hashes), lh)
    got_levels = tree.levels()
    assert len(got_levels) == len(levels)
    for g, w in zip(got_levels, levels):
        assert np.array_equal(bj.to_numpy(g), w)
    assert np.array_equal(tree.get_cap(), capd)
    if n > cap:
        for idx in (0, 1, n // 2 + 3, n - 1):
            leaf, path = tree.get_proof(idx)
            assert O.merkle_verify(leaf, path, capd, idx)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_merkle_chunked_leaves_for_fri_oracles(bj, ctx, k):
    n = 1 << 10
    c0, c1 = O.random_field(rng(k), n), O.random_field(rng(k + 50), n)
    tree = ctx.merkle_tree_construct([bj.to_device(c0), bj.to_device(c1)], 4, elems_per_leaf=k)
    lh = O.merkle_leaf_hashes([c0, c1], elems_per_leaf=k)
    assert np.array_equal(bj.to_numpy(tree.leaf_hashes), lh)
    assert np.array_equal(tree.get_cap(), O.merkle_nodes(lh, 4)[-1])


def test_merkle_lde_layout_coset_major(bj, ctx):
    """witness-oracle shape: LDE of C columns, leaf t = coset*n + row absorbs the C column values at t."""
    log_n, L, C = 8, 4, 9
    a = O.random_field(rng(31), (C, 1 << log_n))
    out = ctx.transform_raw_storages_to_lde(bj.to_device(a), L)           # [C, L, n]
    tree = ctx.merkle_tree_construct([out[c].reshape(-1) for c in range(C)], 16)
    want_lde = O.lde(a, 2)
    lh, levels, cap = O.merkle_tree([want_lde[c].reshape(-1) for c in range(C)], 16)
    assert np.array_equal(bj.to_numpy(tree.leaf_hashes), lh)
    assert np.array_equal(tree.get_cap(), cap)


def test_golden_fixture_leaf_hashes_on_gpu(bj, ctx, golden_fixture):
    """The reference's proof.json: GPU leaf hashes of the opened rows verify against the fixture's caps."""
    c = replay.replay_proof(golden_fixture)  # oracle-side replay (also yields nothing GPU specific)
    assert c["merkle_paths"] > 0
    proof, vk = golden_fixture["proof"], golden_fixture["vk"]
    idxs = _query_indices(golden_fixture)
    for q, idx in zip(proof["queries_per_fri_repetition"], idxs):
        for name, cap in (("witness_query", proof["witness_oracle_cap"]), ("stage_2_query", proof["stage_2_oracle_cap"]),
                          ("quotient_query", proof["quotient_oracle_cap"]), ("setup_query", vk["setup_merkle_tree_cap"])):
            row = np.array(q[name]["leaf_elements"], dtype=np.uint64)[None, :]
            leaf = bj.to_numpy(ctx.poseidon2_hash_rows(bj.to_device(row)))[0]
            path = np.array(q[name]["proof"], dtype=np.uint64).reshape(-1, 4)
            assert O.merkle_verify(leaf, path, np.array(cap, dtype=np.uint64), idx)


def _query_indices(fx):
    vk, proof = fx["vk"], fx["proof"]
    tr = replay.Poseidon2Transcript()
    tr.witness_merkle_tree_cap(vk["setup_merkle_tree_cap"])
    for v in proof["public_inputs"]:
        tr.witness_field_elements([v])
    tr.witness_merkle_tree_cap(proof["witness_oracle_cap"])
    for _ in range(8):
        tr.get_challenge()
    tr.witness_merkle_tree_cap(proof["stage_2_oracle_cap"])
    tr.get_ext_challenge()
    tr.witness_merkle_tree_cap(proof["quotient_oracle_cap"])
    tr.get_ext_challenge()
    for g in ("values_at_z", "values_at_z_omega", "values_at_0"):
        for v in proof[g]:
            tr.witness_field_elements(v["coeffs"])
    tr.get_ext_challenge()
    for cap in [proof["fri_base_oracle_cap"]] + list(proof["fri_intermediate_oracles_caps"]):
        tr.witness_merkle_tree_cap(cap)
        tr.get_ext_challenge()
    tr.witness_field_elements(proof["final_fri_monomials"][0])
    tr.witness_field_elements(proof["final_fri_monomials"][1])
    bb = replay.BoolsBuffer(21)
    out = []
    for _ in proof["queries_per_fri_repetition"]:
        bits = bb.get_bits(tr, 21)
        out.append(sum(b << i for i, b in enumerate(bits)))
    return out


# ------------------------------------------------------------------------------------------- FRI -------
@pytest.mark.parametrize("log_m,log_fold", [(3, 1), (3, 3), (12, 1), (12, 2), (12, 3), (17, 3)])
def test_fri_fold_matches_oracle(bj, ctx, log_m, log_fold):
    m = 1 << log_m
    r = rng(log_m * 4 + log_fold)
    c0, c1 = O.random_field(r, m), O.random_field(r, m)
    alpha = [int(x) for x in O.random_field(r, 2)]
    kappa = O.inv(7)
    o0, o1, new_kappa = ctx.fri_fold(bj.to_device(c0), bj.to_device(c1), log_fold, alpha, kappa)
    roots = O.twiddles(log_m, inverse=True)
    w0, w1, a, k = c0, c1, tuple(alpha), kappa
    for _ in range(log_fold):
        w0, w1 = O.fri_fold(w0, w1, a, roots[: len(w0) // 2], k)
        a = O.ext_mul(a, a)
        k = O.mul(k, k)
    assert np.array_equal(bj.to_numpy(o0), w0) and np.array_equal(bj.to_numpy(o1), w1)
    assert new_kappa == k


def test_fri_fold_golden_fixture(bj, ctx, golden_fixture):
    """Fold the opened FRI leaves of the reference proof on the GPU: the result must be the element found in the
    next oracle's leaf (verifier.rs:2386-2510).  The leaf is embedded at its true position of a zero vector so the
    kernel uses the same root indices as the real codeword."""
    fx = golden_fixture
    c = replay.replay_proof(fx)
    sched = c["schedule"]
    idxs = _query_indices(fx)
    log_full = fx["vk"]["fixed_parameters"]["domain_size"].bit_length() - 1 + 1
    for q, idx in zip(fx["proof"]["queries_per_fri_repetition"][:3], idxs[:3]):
        kappa = O.inv(7)
        sub, log_m = idx, log_full
        for lvl in range(len(sched) - 1):
            k = sched[lvl]
            deg = 1 << k
            tree_idx = sub >> k
            le = q["fri_queries"][lvl]["leaf_elements"]
            c0 = np.zeros(1 << log_m, np.uint64)
            c1 = np.zeros(1 << log_m, np.uint64)
            c0[tree_idx * deg:(tree_idx + 1) * deg] = le[:deg]
            c1[tree_idx * deg:(tree_idx + 1) * deg] = le[deg:]
            alpha = c["challenges"]["fri"][lvl][0]
            o0, o1, kappa = ctx.fri_fold(bj.to_device(c0), bj.to_device(c1), k, alpha, kappa)
            nxt = q["fri_queries"][lvl + 1]["leaf_elements"]
            ndeg = 1 << sched[lvl + 1]
            pos = tree_idx % ndeg
            assert int(bj.to_numpy(o0[tree_idx:tree_idx + 1])[0]) == nxt[pos]
            assert int(bj.to_numpy(o1[tree_idx:tree_idx + 1])[0]) == nxt[ndeg + pos]
            sub, log_m = tree_idx, log_m - k


def test_device_field_selftest(bj, ctx):
    """Inline-PTX mul/add/sub vs the portable C versions inside one kernel (4M random + edge inputs)."""
    import ctypes
    from era_boojum_b200 import native
    bad = ctypes.c_uint64(123)
    st = native.lib.bj_selftest_field(ctx._h, 1 << 22, 20260924, ctypes.byref(bad))
    assert st == 0 and bad.value == 0


# ----------------------------------------------------------------------------- batch inverse / DEEP ---------
@pytest.mark.parametrize("n", [1, 7, 8, 1000, 1 << 16])
def test_batch_inverse_matches_oracle(bj, ctx, n):
    r = rng(n)
    a = O.random_field(r, n)
    a[a == 0] = 1
    got = bj.to_numpy(ctx.batch_inverse_inplace(bj.to_device(a)))
    assert np.array_equal(got, O.batch_inverse(a))
    c0, c1 = O.random_field(r, n), O.random_field(r, n)
    g0, g1 = ctx.batch_inverse_inplace_in_extension(bj.to_device(c0), bj.to_device(c1))
    w0, w1 = O.batch_inverse_ext(c0, c1)
    assert np.array_equal(bj.to_numpy(g0), w0) and np.array_equal(bj.to_numpy(g1), w1)


def test_batch_inverse_zero_maps_to_zero(bj, ctx):
    a = np.array([5, 0, 7, P, 11, 0, 13, 17, 19, 23], dtype=np.uint64)
    got = bj.to_numpy(ctx.batch_inverse_inplace(bj.to_device(a)))
    for x, y in zip(a, got):
        assert int(y) == (pow(int(x) % P, P - 2, P) if int(x) % P else 0)


@pytest.mark.parametrize("log_rows,n_base,n_ext", [(6, 3, 2), (12, 9, 4), (15, 20, 3)])
def test_deep_group_matches_oracle(bj, ctx, log_rows, n_base, n_ext):
    rows = 1 << log_rows
    r = rng(log_rows)
    srcs = [(O.random_field(r, rows), None) for _ in range(n_base)]
    srcs += [(O.random_field(r, rows), O.random_field(r, rows)) for _ in range(n_ext)]
    n = len(srcs)
    vals = [tuple(int(x) for x in O.random_field(r, 2)) for _ in range(n)]
    for i in range(n_base):
        vals[i] = (vals[i][0], vals[i][1])  # the value at an Fp2 point is in Fp2 even for base-field polynomials
    chs = [tuple(int(x) for x in O.random_field(r, 2)) for _ in range(n)]
    acc0, acc1 = O.random_field(r, rows), O.random_field(r, rows)
    for at in ([int(x) for x in O.random_field(r, 2)], [0, 0], [int(O.omega(4)), 0]):
        d_srcs = [(bj.to_device(s0), bj.to_device(s1) if s1 is not None else None) for s0, s1 in srcs]
        g0, g1 = ctx.quotening_operation_in_extension(bj.to_device(acc0), bj.to_device(acc1), d_srcs, vals, at, chs)
        w0, w1 = O.deep_group(acc0, acc1, srcs, vals, chs, at)
        assert np.array_equal(bj.to_numpy(g0), w0) and np.array_equal(bj.to_numpy(g1), w1)


def test_deep_golden_fixture_point(bj, ctx, golden_fixture):
    """One opened row of the reference proof embedded at its true LDE position: the GPU DEEP value over the four
    opening groups equals the element in the first FRI leaf (verifier.rs:2154-2384)."""
    fx = golden_fixture
    c = replay.replay_proof(fx)
    proof, vk = fx["proof"], fx["vk"]
    fp = vk["fixed_parameters"]
    log_n = fp["domain_size"].bit_length() - 1
    log_rows = log_n + 1
    idx = _query_indices(fx)[0]
    q = proof["queries_per_fri_repetition"][0]
    wq, sq = q["witness_query"]["leaf_elements"], q["stage_2_query"]["leaf_elements"]
    qq, uq = q["quotient_query"]["leaf_elements"], q["setup_query"]["leaf_elements"]
    V, C, vw = 155, 8, 155
    base = lambda els: [(e, None) for e in els]
    ext = lambda els: [(els[i], els[i + 1]) for i in range(0, len(els), 2)]
    src_z = base(wq[:vw]) + base(uq[V:V + C]) + base(uq[:V]) + ext(sq[0:2]) + ext(sq[2:40]) + base(wq[vw:vw + 1]) \
        + ext(sq[40:56]) + ext(sq[56:]) + base(uq[V + C:V + C + 4]) + ext(qq)
    groups = [(src_z, [tuple(v["coeffs"]) for v in proof["values_at_z"]], c["challenges"]["z"])]
    w_n = replay.omega(log_n)
    z = c["challenges"]["z"]
    groups.append((ext(sq[0:2]), [tuple(v["coeffs"]) for v in proof["values_at_z_omega"]], replay.e_mul_base(z, w_n)))
    groups.append((ext(sq[40:56]) + ext(sq[56:]), [tuple(v["coeffs"]) for v in proof["values_at_0"]], (0, 0)))
    pi_at = pow(w_n, fp["public_inputs_locations"][0][1], P)
    groups.append(([(wq[col], None) for col, _ in fp["public_inputs_locations"]],
                   [(v, 0) for v in proof["public_inputs"]], (pi_at, 0)))
    ch = replay.ext_powers(c["challenges"]["deep"], 374)
    import torch
    acc0 = torch.zeros(1 << log_rows, dtype=torch.int64, device="cuda:0")
    acc1 = torch.zeros(1 << log_rows, dtype=torch.int64, device="cuda:0")
    off = 0
    for srcs, vals, at in groups:
        d_srcs = []
        for s0, s1 in srcs:
            t0 = torch.zeros(1 << log_rows, dtype=torch.int64, device="cuda:0")
            t0[idx] = int(np.array([s0], dtype=np.uint64).view(np.int64)[0])
            t1 = None
            if s1 is not None:
                t1 = torch.zeros(1 << log_rows, dtype=torch.int64, device="cuda:0")
                t1[idx] = int(np.array([s1], dtype=np.uint64).view(np.int64)[0])
            d_srcs.append((t0, t1))
        ctx.quotening_operation_in_extension(acc0, acc1, d_srcs, vals, at, ch[off:off + len(srcs)])
        off += len(srcs)
        del d_srcs
    assert off == 374
    le = q["fri_queries"][0]["leaf_elements"]
    sub = idx % 8
    got = (int(bj.to_numpy(acc0[idx:idx + 1])[0]), int(bj.to_numpy(acc1[idx:idx + 1])[0]))
    assert got == (le[sub], le[8 + sub])


# ------------------------------------------------------------------------------ gate / quotient evaluator -----
def _sha_gate_programs():
    """The SSA programs gpu_synthesizer::GPUDataCapture::from_evaluator records for the three evaluators of the
    SHA-256 bench circuit (src/gadgets/sha256/mod.rs:348-373), written out by hand."""
    from era_boojum_b200 import native as N
    V, C, CS, T = N.IDX_VARIABLE, N.IDX_CONSTANT_POLY, N.IDX_CONSTANT_POLY_SHARED, N.IDX_TEMPORARY
    fma = dict(relations=[(N.REL_MUL, 0, (V, 2), (CS, 1)),      # contribution = c * linear_coeff
                          (N.REL_MUL, 1, (V, 0), (V, 1)),       # t = a * b
                          (N.REL_MUL, 2, (CS, 0), (T, 1)),      # quad * t
                          (N.REL_ADD, 3, (T, 0), (T, 2)),
                          (N.REL_SUB, 4, (T, 3), (V, 3))],
               writes=[(T, 4)], variables_offset=4, constants_offset=0)
    red = dict(relations=[(N.REL_MUL, 0, (V, 0), (CS, 0)), (N.REL_MUL, 1, (V, 1), (CS, 1)), (N.REL_ADD, 2, (T, 0), (T, 1)),
                          (N.REL_MUL, 3, (V, 2), (CS, 2)), (N.REL_ADD, 4, (T, 2), (T, 3)),
                          (N.REL_MUL, 5, (V, 3), (CS, 3)), (N.REL_ADD, 6, (T, 4), (T, 5)),
                          (N.REL_SUB, 7, (T, 6), (V, 4))],
               writes=[(T, 7)], variables_offset=5, constants_offset=0)
    ca = dict(relations=[(N.REL_SUB, 0, (V, 0), (C, 0))], writes=[(T, 0)], variables_offset=1, constants_offset=1)
    return {"fma": fma, "reduction4": red, "constant_allocator": ca}


@pytest.mark.parametrize("log_rows", [5, 11])
def test_gate_evaluator_sha_circuit_shape(bj, ctx, log_rows):
    """60 general-purpose columns, 4 + 3 constant columns, gates ConstantAllocator x4 / FMA x15 / Reduction<4> x12 with
    selector paths of a 3-level tree; compared point by point with the oracle's restatement of the reference."""
    from oracle import gates as G
    rows = 1 << log_rows
    r = rng(log_rows)
    n_vars, n_consts = 60, 7
    var_cols = [O.random_field(r, rows) for _ in range(n_vars)]
    const_cols = [O.random_field(r, rows) for _ in range(n_consts)]
    layout = [("constant_allocator", 4, [True, False]), ("fma", 15, [True, True]), ("reduction4", 12, [False])]
    n_terms = sum(reps for _, reps, _ in layout)
    alphas = [tuple(int(x) for x in O.random_field(r, 2)) for _ in range(n_terms)]
    progs = _sha_gate_programs()
    gates = []
    for name, reps, path in layout:
        g = dict(progs[name])
        g.update(num_repetitions=reps, constants_placement_offset=len(path), selector_path=path)
        gates.append(g)
    q0, q1 = O.random_field(r, rows), O.random_field(r, rows)
    d0, d1 = bj.to_device(q0), bj.to_device(q1)
    ctx.evaluate_gates_over_general_purpose_columns(gates, [bj.to_device(c) for c in var_cols], [],
                                                    [bj.to_device(c) for c in const_cols], alphas, d0, d1)
    g0, g1 = bj.to_numpy(d0), bj.to_numpy(d1)
    check = range(rows) if rows <= 64 else list(range(0, rows, 37)) + [rows - 1]
    for t in check:
        vr = [int(c[t]) for c in var_cols]
        cr = [int(c[t]) for c in const_cols]
        w0, w1 = G.quotient_gates_row(layout, vr, cr, alphas)
        assert int(g0[t]) == (int(q0[t]) + w0) % P and int(g1[t]) == (int(q1[t]) + w1) % P, t


def test_gate_evaluator_all_relations(bj, ctx):
    """every Relation kind incl. Double / Negate / Square / Inverse, witness columns and immediate constants."""
    from era_boojum_b200 import native as N
    rows = 256
    r = rng(3)
    v = [O.random_field(r, rows) for _ in range(2)]
    w = [O.random_field(r, rows)]
    w[0][w[0] == 0] = 1
    c = [O.random_field(r, rows)]
    V, W, C, T, K = N.IDX_VARIABLE, N.IDX_WITNESS, N.IDX_CONSTANT_POLY, N.IDX_TEMPORARY, N.IDX_CONSTANT_VALUE
    rel = [(N.REL_DOUBLE, 0, (V, 0), None), (N.REL_NEGATE, 1, (V, 1), None), (N.REL_SQUARE, 2, (T, 0), None),
           (N.REL_INVERSE, 3, (W, 0), None), (N.REL_MUL, 4, (T, 2), (T, 3)), (N.REL_ADD, 5, (T, 4), (K, 12345)),
           (N.REL_SUB, 6, (T, 5), (C, 0)), (N.REL_MUL, 7, (T, 6), (T, 1))]
    gate = dict(relations=rel, writes=[(T, 7), (T, 1)], num_repetitions=1, constants_placement_offset=0, selector_path=[])
    alphas = [(3, 5), (7, 11)]
    import torch
    d0 = torch.zeros(rows, dtype=torch.int64, device="cuda:0")
    d1 = torch.zeros(rows, dtype=torch.int64, device="cuda:0")
    ctx.evaluate_gates_over_general_purpose_columns([gate], [bj.to_device(x) for x in v], [bj.to_device(x) for x in w],
                                                    [bj.to_device(x) for x in c], alphas, d0, d1)
    g0, g1 = bj.to_numpy(d0), bj.to_numpy(d1)
    for t in range(rows):
        a, b, ww, cc = int(v[0][t]), int(v[1][t]), int(w[0][t]), int(c[0][t])
        t1 = (-b) % P
        t7 = ((((2 * a) ** 2 % P) * pow(ww, P - 2, P) + 12345 - cc) % P) * t1 % P
        assert int(g0[t]) == (t7 * 3 + t1 * 7) % P and int(g1[t]) == (t7 * 5 + t1 * 11) % P


def test_gate_programs_of_the_reference_fixture_circuit(bj, ctx, golden_fixture):
    """The gate set the reference verifies proof.json with (recursive_verifier.rs:2290-2368; the 13 gate types of
    gpu_synthesizer/mod.rs:826-838 minus the two this circuit does not use), as recorded SSA programs through
    bj_quotient_gates_general_purpose: 11 evaluators over 130 general-purpose columns with the vk's own selector tree (the
    Poseidon2 flattened gate alone is ~9k relations, 118 terms) plus the boolean gate over a specialised column, against the
    same evaluators run over the base field (oracle/verifier_reference.py, pinned by the quotient identity on proof.json)."""
    from era_boojum_b200 import gate_library as GL
    from era_boojum_b200 import placement as PL
    from oracle import verifier_reference as VR
    fp = golden_fixture["vk"]["fixed_parameters"]
    cfg = VR.REFERENCE_FIXTURE_GATES
    lay = VR.circuit_layout(fp, cfg)
    rows = 96
    r = rng(1300)
    V, C = lay["num_variables"], lay["num_constants"]
    var_cols = [r.integers(0, 2**64, size=rows, dtype=np.uint64) for _ in range(V)]      # non-canonical values included
    const_cols = [O.random_field(r, rows) for _ in range(C)]
    tree = fp["selectors_placement"]
    gates, plan = [], []
    for s_ in lay["specialized"]:                               # specialised-column gates come first (prover.rs:608-625)
        gates.append(GL.placed(s_["gate"], s_["reps"], [], constants_placement_offset=lay["consts_gp"] + s_["const_base"],
                               variables_initial_offset=s_["var_base"]))
        plan.append((s_["gate"], s_["reps"], [], s_["var_base"], lay["consts_gp"] + s_["const_base"]))
    for gate_idx, gate in enumerate(cfg["general_purpose"]):
        if gate.terms == 0:
            continue
        reps = gate.num_repetitions_in_geometry(lay["gp_vars"], 0, fp["parameters"]["num_constant_columns"])
        path = PL.output_placement(tree, gate_idx)
        gates.append(GL.placed(gate, reps, path))
        plan.append((gate, reps, path, 0, len(path)))
    n_terms = sum(g.terms * reps for g, reps, *_ in plan)
    assert n_terms == 415
    alphas = [tuple(int(x) for x in O.random_field(r, 2)) for _ in range(n_terms)]
    q0, q1 = O.random_field(r, rows), O.random_field(r, rows)
    d0, d1 = bj.to_device(q0), bj.to_device(q1)
    ctx.evaluate_gates_over_general_purpose_columns(gates, [bj.to_device(c) for c in var_cols], [],
                                                    [bj.to_device(c) for c in const_cols], alphas, d0, d1)
    g0, g1 = bj.to_numpy(d0), bj.to_numpy(d1)
    B = VR.BaseBackend
    for t in list(range(0, rows, 7)) + [rows - 1]:
        vr = [int(c[t]) % P for c in var_cols]
        cr = [int(c[t]) for c in const_cols]
        w0 = w1 = k = 0
        for gate, reps, path, var_base, const_base in plan:
            terms = GL.evaluate_gate_terms(gate, B, lambda i: vr[i], lambda i: 0, lambda i: cr[i], reps, var_base=var_base,
                                           const_base=const_base)
            sel = 1
            for depth, bit in enumerate(path):
                sel = sel * (cr[depth] if bit else (1 - cr[depth])) % P
            a0 = a1 = 0
            for term in terms:
                a0, a1, k = (a0 + term * alphas[k][0]) % P, (a1 + term * alphas[k][1]) % P, k + 1
            w0, w1 = (w0 + sel * a0) % P, (w1 + sel * a1) % P
        assert int(g0[t]) == (int(q0[t]) + w0) % P and int(g1[t]) == (int(q1[t]) + w1) % P, t
    # the interpreter handles 1, 2 or 4 points per thread (chosen by size; forced here): same result, incl. the ragged tail
    # (96 rows = not a multiple of the 256- / 512-point blocks)
    for k in (1, 2, 4):
        os.environ["BJ_GATE_POINTS_PER_THREAD"] = str(k)
        try:
            ck = bj.Context(0)
        finally:
            del os.environ["BJ_GATE_POINTS_PER_THREAD"]
        e0, e1 = bj.to_device(q0), bj.to_device(q1)
        ck.evaluate_gates_over_general_purpose_columns(gates, [bj.to_device(c) for c in var_cols], [],
                                                       [bj.to_device(c) for c in const_cols], alphas, e0, e1)
        ck.synchronize()
        assert np.array_equal(bj.to_numpy(e0), g0) and np.array_equal(bj.to_numpy(e1), g1), k
        ck.close()
    # the host peephole (x * 1, x + 0 aliases; multiply-add fusion) changes the program, not the values: all settings agree (15 = default: aliases, multiply-add fusion, linear combinations, pushing steps)
    for mode in (0, 1, 3, 7, 13):
        os.environ["BJ_GATE_PEEPHOLE"] = str(mode)
        try:
            ck = bj.Context(0)
        finally:
            del os.environ["BJ_GATE_PEEPHOLE"]
        e0, e1 = bj.to_device(q0), bj.to_device(q1)
        ck.evaluate_gates_over_general_purpose_columns(gates, [bj.to_device(c) for c in var_cols], [],
                                                       [bj.to_device(c) for c in const_cols], alphas, e0, e1)
        ck.synchronize()
        assert np.array_equal(bj.to_numpy(e0), g0) and np.array_equal(bj.to_numpy(e1), g1), mode
        ck.close()


def test_gate_program_limits(bj, ctx):
    """a program may name 2^20 temporaries, but at most 128 may be live at once; programs must be SSA."""
    import torch
    from era_boojum_b200 import native as N
    V, T, K = N.IDX_VARIABLE, N.IDX_TEMPORARY, N.IDX_CONSTANT_VALUE
    rows = 32
    v = [bj.to_device(O.random_field(rng(2), rows))]
    d0 = torch.zeros(rows, dtype=torch.int64, device="cuda:0")
    d1 = torch.zeros(rows, dtype=torch.int64, device="cuda:0")
    # 200 temporaries all kept alive until the end -> unsupported
    rel = [(N.REL_ADD, i, (V, 0), (K, i)) for i in range(200)]
    rel += [(N.REL_ADD, 200 + i, (T, i), (T, 199 - i)) for i in range(200)]
    gate = dict(relations=rel, writes=[(T, 399)], num_repetitions=1, constants_placement_offset=0, selector_path=[])
    with pytest.raises(bj.BoojumError) as e:
        ctx.evaluate_gates_over_general_purpose_columns([gate], v, [], [], [(1, 0)], d0, d1)
    assert e.value.status == N.BJ_ERR_UNSUPPORTED
    # a chain of 5000 relations with two live temporaries is fine: x + 5000
    rel = [(N.REL_ADD, 0, (V, 0), (K, 1))] + [(N.REL_ADD, i, (T, i - 1), (K, 1)) for i in range(1, 5000)]
    gate = dict(relations=rel, writes=[(T, 4999)], num_repetitions=1, constants_placement_offset=0, selector_path=[])
    ctx.evaluate_gates_over_general_purpose_columns([gate], v, [], [], [(1, 0)], d0, d1)
    assert np.array_equal(bj.to_numpy(d0), (bj.to_numpy(v[0]).astype(object) + 5000) % P)
    # not SSA (temporary 0 defined twice)
    gate = dict(relations=[(N.REL_ADD, 0, (V, 0), (K, 1)), (N.REL_ADD, 0, (V, 0), (K, 2))], writes=[(T, 0)], num_repetitions=1,
                constants_placement_offset=0, selector_path=[])
    with pytest.raises(bj.BoojumError):
        ctx.evaluate_gates_over_general_purpose_columns([gate], v, [], [], [(1, 0)], d0, d1)


# --------------------------------------------------------------------------------------- do_fri / queries -----
@pytest.mark.parametrize("log_n,log_lde,cap,schedule", [(8, 3, 16, [3, 3, 1]), (10, 1, 4, [3, 3, 2]), (12, 3, 16, [3, 3, 3, 2])])
def test_do_fri_matches_oracle_and_verifies(bj, ctx, log_n, log_lde, cap, schedule):
    """Commit phase on the GPU (host transcript in C++) == the oracle's do_fri: caps, challenges, final monomials;
    then queries answered by the library verify with the reference verifier's FRI chain (verifier.rs:2386-2510)."""
    n, L = 1 << log_n, 1 << log_lde
    r = rng(log_n * 7 + log_lde)
    m = O.random_field(r, (2, n))                      # two monomial forms: the c0 / c1 parts of a degree < n Fp2 polynomial
    lde = O.lde(m, log_lde, from_monomials=True)       # [2, L, n]
    c0, c1 = lde[0].reshape(-1), lde[1].reshape(-1)
    seed_els = [int(x) for x in O.random_field(r, 5)]
    t_ref = replay.Poseidon2Transcript()
    t_ref.witness_field_elements(seed_els)
    want = replay.do_fri_oracle(c0, c1, t_ref, schedule, log_lde, cap)
    t_gpu = bj.Transcript()
    t_gpu.witness_field_elements(seed_els)
    d0, d1 = bj.to_device(c0), bj.to_device(c1)
    fo = ctx.do_fri(t_gpu, d0, d1, schedule, L, cap)
    assert fo.num_oracles() == len(schedule)
    for i in range(len(schedule)):
        assert np.array_equal(fo.get_cap(i), want["caps"][i])
    assert fo.challenges() == [tuple(int(x) for x in a) for a in want["challenges"]]
    g0, g1 = fo.monomial_forms()
    assert np.array_equal(g0, want["monomials"][0]) and np.array_equal(g1, want["monomials"][1])
    # both transcripts are in the same state afterwards
    assert t_gpu.get_challenge() == t_ref.get_challenge()
    # queries
    for idx in [0, 1, (n * L) // 3, n * L - 1]:
        qs, sub = [], idx
        for lvl, k in enumerate(schedule):
            le, path = fo.query(lvl, sub >> k, k)
            qs.append((le, path))
            sub >>= k
        assert replay.verify_fri_query(idx, log_n, log_lde, schedule, cap, [fo.get_cap(i) for i in range(len(schedule))],
                                       fo.challenges(), (g0, g1), qs, start_value=(int(c0[idx]), int(c1[idx])))


def test_do_fri_rejects_high_degree(bj, ctx):
    r = rng(99)
    c0, c1 = O.random_field(r, 1 << 9), O.random_field(r, 1 << 9)   # random codeword: not an LDE
    with pytest.raises(bj.BoojumError):
        ctx.do_fri(bj.Transcript(), bj.to_device(c0), bj.to_device(c1), [3, 2], 8, 4)


def test_query_helpers_match_oracle(bj, ctx):
    n, C, cap = 1 << 9, 13, 8
    cols = [O.random_field(rng(c), n) for c in range(C)]
    d_cols = [bj.to_device(c) for c in cols]
    tree = ctx.merkle_tree_construct(d_cols, cap)
    lh, levels, capd = O.merkle_tree(cols, cap)
    idx = [0, 5, 77, n - 1]
    rows = ctx.query_leaf_elements(d_cols, idx)
    paths = ctx.merkle_paths(tree, idx)
    for q, i in enumerate(idx):
        assert np.array_equal(rows[q], np.array([c[i] for c in cols], dtype=np.uint64))
        assert np.array_equal(paths[q], O.merkle_path(lh, levels, i))
        assert O.merkle_verify(O.poseidon2_hash_leaf(rows[q]), paths[q], capd, i)


def test_merkle_full_size_config3_paths_verify_against_cap(bj, ctx):
    """BASELINE config 3 (2^22 leaves x 100 columns, cap 16): the oracle cannot rebuild the tree in seconds, so the full-size
    check is the size-independent one - 192 random leaves are re-hashed by the oracle from the opened rows and their paths
    must lead to the cap the GPU produced (a wrong node anywhere on those paths, or a wrong leaf hash, breaks it)."""
    import torch
    log_leaves, n_cols, cap = 22, 100, 16
    gen = torch.Generator(device="cuda:0")
    gen.manual_seed(7)
    d_cols = [torch.randint(0, 2**63 - 1, (1 << log_leaves,), dtype=torch.int64, device="cuda:0", generator=gen) for _ in range(n_cols)]
    tree = ctx.merkle_tree_construct(d_cols, cap)
    capd = tree.get_cap()
    assert capd.shape == (cap, 4) and len({tuple(r) for r in capd.tolist()}) == cap
    idx = [0, (1 << log_leaves) - 1] + [int(v) for v in rng(5).integers(0, 1 << log_leaves, 190)]
    rows = ctx.query_leaf_elements(d_cols, idx)
    paths = ctx.merkle_paths(tree, idx)
    assert paths.shape[1] == log_leaves - 4
    for q, i in enumerate(idx):
        assert O.merkle_verify(O.poseidon2_hash_leaf(rows[q]), paths[q], capd, i), i
    # a flipped bit in an opened row must not verify
    bad = rows[0].copy()
    bad[37] ^= 1
    assert not O.merkle_verify(O.poseidon2_hash_leaf(bad), paths[0], capd, idx[0])


# ------------------------------------------------------------------------------------ stage 2 (copy permutation) -----
def _satisfying_copy_permutation(r, n_cols, log_n):
    """variable columns with repeated values and sigma columns encoding the cycles of equal cells
    (sigma_j[i] = k_j' * omega^i' of the next cell in the cycle; identity for untouched cells)."""
    from oracle import stage2 as S
    n = 1 << log_n
    ks = S.non_residues_for_copy_permutation(n, n_cols)
    w_n = replay.omega(log_n)
    vals = [[int(x) for x in O.random_field(r, n)] for _ in range(n_cols)]
    sig = [[ks[j] * pow(w_n, i, P) % P for i in range(n)] for j in range(n_cols)]
    cells = [(j, i) for j in range(n_cols) for i in range(n)]
    perm = r.permutation(len(cells))
    for g in range(0, len(cells) - 2, 3):           # cycles of three cells sharing one value
        cyc = [cells[perm[g + t]] for t in range(3)]
        v = vals[cyc[0][0]][cyc[0][1]]
        for (j, i), (j2, i2) in zip(cyc, cyc[1:] + cyc[:1]):
            vals[j][i] = v
            sig[j][i] = ks[j2] * pow(w_n, i2, P) % P
    return vals, sig


@pytest.mark.parametrize("n_cols,log_n,deg", [(3, 4, 4), (9, 5, 4), (7, 6, 2), (5, 12, 2)])
def test_copy_permutation_stage2_matches_oracle(bj, ctx, n_cols, log_n, deg):
    from oracle import stage2 as S
    r = rng(n_cols * 10 + log_n)
    vals, sig = _satisfying_copy_permutation(r, n_cols, log_n)
    beta = tuple(int(x) for x in O.random_field(r, 2))
    gamma = tuple(int(x) for x in O.random_field(r, 2))
    d_v = [bj.to_device(np.array(c, dtype=np.uint64)) for c in vals]
    d_s = [bj.to_device(np.array(c, dtype=np.uint64)) for c in sig]
    z0, z1, partials = ctx.compute_partial_products_in_extension(d_v, d_s, beta, gamma, deg)
    g0, g1 = bj.to_numpy(z0), bj.to_numpy(z1)
    if log_n <= 6:
        wz, wp = S.partial_products(vals, sig, beta, gamma, deg)
        assert [(int(a), int(b)) for a, b in zip(g0, g1)] == wz
        assert len(partials) == len(wp)
        for (p0, p1), w in zip(partials, wp):
            assert [(int(a), int(b)) for a, b in zip(bj.to_numpy(p0), bj.to_numpy(p1))] == w
    else:
        # large domain: z[0] = 1 and the defining recurrence z[i+1] = z[i] * prod_j num_j / den_j at sampled rows
        assert (int(g0[0]), int(g1[0])) == (1, 0)
        ks = S.non_residues_for_copy_permutation(1 << log_n, n_cols)
        w_n = replay.omega(log_n)
        for i in [0, 1, 77, 2047, (1 << log_n) - 2]:
            x = pow(w_n, i, P)
            num, den = (1, 0), (1, 0)
            for j in range(n_cols):
                w = vals[j][i]
                num = replay.e_mul(num, replay.e_add(replay.e_add(replay.e_mul_base(beta, ks[j] * x % P), (w, 0)), gamma))
                den = replay.e_mul(den, replay.e_add(replay.e_add(replay.e_mul_base(beta, sig[j][i]), (w, 0)), gamma))
            lhs = replay.e_mul((int(g0[i + 1]), int(g1[i + 1])), den)
            assert lhs == replay.e_mul((int(g0[i]), int(g1[i])), num)


def test_copy_permutation_rejects_unsatisfied(bj, ctx):
    r = rng(4)
    vals, sig = _satisfying_copy_permutation(r, 3, 5)
    vals[1][7] = (vals[1][7] + 1) % P   # break one copy constraint (cell is in a cycle with overwhelming probability)
    broken = any(sig[1][7] != v for v in [0])
    d_v = [bj.to_device(np.array(c, dtype=np.uint64)) for c in vals]
    d_s = [bj.to_device(np.array(c, dtype=np.uint64)) for c in sig]
    from oracle import stage2 as S
    ks = S.non_residues_for_copy_permutation(32, 3)
    if sig[1][7] == ks[1] * pow(replay.omega(5), 7, P) % P:
        pytest.skip("cell happened to be untouched")
    with pytest.raises(bj.BoojumError):
        ctx.compute_partial_products_in_extension(d_v, d_s, (3, 4), (5, 6), 2)


# ----------------------------------------------------------------------------- openings / quotient pieces -----
@pytest.mark.parametrize("log_n,n_cols", [(3, 2), (8, 11), (13, 20)])
def test_barycentric_evaluate_matches_horner(bj, ctx, log_n, n_cols):
    from oracle import stage2 as S
    r = rng(log_n + n_cols)
    vals = O.random_field(r, (n_cols, 1 << log_n))
    mono = O.intt_n2n(vals)
    lde = ctx.transform_raw_storages_to_lde(bj.to_device(vals), 2)
    cols = [lde[c].reshape(-1) for c in range(n_cols)]
    for at in (tuple(int(x) for x in O.random_field(r, 2)), (0, 0), (int(O.omega(log_n + 1)), 0)):
        got = ctx.barycentric_evaluate(cols, log_n, at)
        for c in range(0, n_cols, max(1, n_cols // 5)):
            assert got[c] == S.horner_ext(mono[c], at)


def test_quotient_copy_permutation_and_vanishing_match_oracle(bj, ctx):
    from oracle import stage2 as S
    log_n, log_lde, log_q, n_cols, chunk = 5, 3, 2, 5, 2
    r = rng(55)
    vals, sig = _satisfying_copy_permutation(r, n_cols, log_n)
    beta = tuple(int(x) for x in O.random_field(r, 2))
    gamma = tuple(int(x) for x in O.random_field(r, 2))
    v_np = np.array(vals, dtype=np.uint64)
    s_np = np.array(sig, dtype=np.uint64)
    d_v, d_s = bj.to_device(v_np), bj.to_device(s_np)
    z0, z1, partials = ctx.compute_partial_products_in_extension([d_v[c] for c in range(n_cols)], [d_s[c] for c in range(n_cols)],
                                                                 beta, gamma, chunk)
    L = 1 << log_lde
    lde_v = ctx.transform_raw_storages_to_lde(d_v, L)
    lde_s = ctx.transform_raw_storages_to_lde(d_s, L)
    import torch
    st2 = torch.stack([z0, z1] + [t for pr in partials for t in pr])
    lde_2 = ctx.transform_raw_storages_to_lde(st2.contiguous(), L)
    flat = lambda t: t.reshape(-1)
    n_chunks = (n_cols + chunk - 1) // chunk
    alphas = [tuple(int(x) for x in O.random_field(r, 2)) for _ in range(n_chunks + 1)]
    npts = 1 << (log_n + log_q)
    q0 = torch.zeros(npts, dtype=torch.int64, device="cuda:0")
    q1 = torch.zeros(npts, dtype=torch.int64, device="cuda:0")
    part_ldes = [(flat(lde_2[2 + 2 * c]), flat(lde_2[3 + 2 * c])) for c in range(n_chunks - 1)]
    ctx.quotient_copy_permutation([flat(lde_v[c]) for c in range(n_cols)], [flat(lde_s[c]) for c in range(n_cols)],
                                  (flat(lde_2[0]), flat(lde_2[1])), part_ldes, beta, gamma, alphas, log_n, log_lde, log_q, chunk,
                                  q0, q1)
    g0, g1 = bj.to_numpy(q0), bj.to_numpy(q1)
    hv, hs, h2 = bj.to_numpy(lde_v).reshape(n_cols, -1), bj.to_numpy(lde_s).reshape(n_cols, -1), bj.to_numpy(lde_2).reshape(2 * n_chunks, -1)
    hz = (h2[0], h2[1])
    hp = [(h2[2 + 2 * c], h2[3 + 2 * c]) for c in range(n_chunks - 1)]
    for t in list(range(0, npts, 7)) + [npts - 1]:
        want = S.quotient_copy_permutation_point(t, log_n, log_lde, hv, hs, hz, hp, beta, gamma, alphas, chunk)
        assert (int(g0[t]), int(g1[t])) == want, t
    ctx.divide_by_vanishing(q0, q1, log_n, log_q)
    d0, d1 = bj.to_numpy(q0), bj.to_numpy(q1)
    for t in (0, 33, 100, npts - 1):
        vi = S.vanishing_inverse(log_n, log_q, t >> log_n)
        assert int(d0[t]) == int(g0[t]) * vi % P and int(d1[t]) == int(g1[t]) * vi % P
    # the quotient restricted to these terms is a polynomial of degree < n*Q: after un-bit-reversing and an iNTT on
    # coset 7 of size n*Q the top quarter of the coefficients is not constrained, but the value must re-evaluate:
    # cheap check instead: the relation terms vanish on the trace domain => division produced no poles; verified by
    # re-multiplying and comparing with the undivided values above.


# ------------------------------------------------------------------------------------------- lookup argument -----
@pytest.mark.parametrize("n_sub,width,with_id", [(1, 1, False), (3, 4, True), (8, 4, True), (2, 3, False)])
def test_lookup_polys_and_quotient_terms_match_oracle(bj, ctx, n_sub, width, with_id):
    """bj_lookup_polys_specialized / bj_quotient_lookup_specialized against the Python-int restatement of
    lookup_argument_in_ext.rs:320-947 and :949-1319 (oracle/lookup.py) on random columns: the formulas are pointwise, so
    no satisfying assignment is needed for parity (non-canonical inputs included)."""
    import torch
    from oracle import lookup as LK
    log_n, log_lde, log_q = 5, 3, 2
    n = 1 << log_n
    r = rng(100 * n_sub + width)
    n_tab = width + (1 if with_id else 0)
    cols = r.integers(0, 2**64, size=(n_sub * width, n), dtype=np.uint64)
    tid = r.integers(0, 2**64, size=n, dtype=np.uint64) if with_id else None
    tabs = O.random_field(r, (n_tab, n))
    mult = O.random_field(r, n)
    beta = tuple(int(x) for x in O.random_field(r, 2))
    gamma = tuple(int(x) for x in O.random_field(r, 2))
    d_cols, d_tabs, d_mult = bj.to_device(cols), bj.to_device(tabs), bj.to_device(mult)
    d_tid = bj.to_device(tid) if with_id else None
    A, B = ctx.compute_lookup_poly_pairs_specialized([d_cols[i] for i in range(n_sub * width)], width, d_tid,
                                                     [d_tabs[i] for i in range(n_tab)], d_mult, beta, gamma)
    wA, wB = LK.lookup_polys(list(cols), width, tid, list(tabs), mult, beta, gamma)
    for i in range(n_sub):
        g0, g1 = bj.to_numpy(A[i][0]), bj.to_numpy(A[i][1])
        assert [(int(a), int(b)) for a, b in zip(g0, g1)] == wA[i], i
    g0, g1 = bj.to_numpy(B[0]), bj.to_numpy(B[1])
    assert [(int(a), int(b)) for a, b in zip(g0, g1)] == wB

    # quotient terms on the first Q*n points of LDE columns (the kernel is pointwise: random "LDE" columns suffice)
    npts = n << log_q
    full = n << log_lde
    L_cols = r.integers(0, 2**64, size=(n_sub * width, full), dtype=np.uint64)
    L_tid = O.random_field(r, full) if with_id else None
    L_tabs = O.random_field(r, (n_tab, full))
    L_mult = O.random_field(r, full)
    L_a = O.random_field(r, (n_sub, 2, full))
    L_b = O.random_field(r, (2, full))
    alphas = [tuple(int(x) for x in O.random_field(r, 2)) for _ in range(n_sub + 1)]
    dc, dt, dm, da, db = (bj.to_device(x) for x in (L_cols, L_tabs, L_mult, L_a, L_b))
    dtid = bj.to_device(L_tid) if with_id else None
    init = O.random_field(r, (2, npts))                      # the kernel ACCUMULATES into q
    dq = bj.to_device(init)
    ctx.quotient_lookup_specialized([dc[i] for i in range(n_sub * width)], width, dtid, [dt[i] for i in range(n_tab)], dm,
                                    [(da[i, 0], da[i, 1]) for i in range(n_sub)], (db[0], db[1]), beta, gamma, alphas, dq[0], dq[1])
    got = bj.to_numpy(dq)
    for t in list(range(0, npts, 5)) + [npts - 1]:
        term = LK.quotient_lookup_point(t, list(L_cols), width, L_tid, list(L_tabs), L_mult,
                                        [(L_a[i, 0], L_a[i, 1]) for i in range(n_sub)], (L_b[0], L_b[1]), beta, gamma, alphas)
        want = ((int(init[0][t]) + term[0]) % P, (int(init[1][t]) + term[1]) % P)
        assert (int(got[0][t]), int(got[1][t])) == want, t


# ------------------------------------------------------------------------------------------- Blake2s tree -----
def _blake2s_leaf(vals):
    import hashlib
    return hashlib.blake2s(b"".join(int(v % P).to_bytes(8, "little") for v in vals), digest_size=32).digest()


@pytest.mark.parametrize("n_cols,log_leaves,cap,epl", [(1, 3, 1, 1), (8, 5, 4, 1), (9, 6, 8, 1), (93, 8, 16, 1), (2, 6, 4, 8)])
def test_merkle_blake2s_matches_hashlib(bj, ctx, n_cols, log_leaves, cap, epl):
    """oracle: CPython hashlib.blake2s (RFC 7693 reference implementation) - the algorithm the `blake2` crate implements."""
    import hashlib
    n = 1 << log_leaves
    r = rng(n_cols + log_leaves)
    cols = [r.integers(0, 2**64, size=n * epl, dtype=np.uint64) for _ in range(n_cols)]   # includes non-canonical values
    tree = ctx.merkle_tree_construct([bj.to_device(c) for c in cols], cap, elems_per_leaf=epl, hasher="blake2s")
    lh = bj.to_numpy(tree.leaf_hashes)
    want = []
    for m in range(n):
        pre = [int(c[m * epl + e]) for c in cols for e in range(epl)]
        want.append(_blake2s_leaf(pre))
    for m in range(n):
        assert lh[m].tobytes() == want[m], m
    level = want
    for got in tree.levels():
        level = [hashlib.blake2s(level[2 * i] + level[2 * i + 1], digest_size=32).digest() for i in range(len(level) // 2)]
        g = bj.to_numpy(got)
        assert [g[i].tobytes() for i in range(len(level))] == level
    assert len(level) == cap


def test_blake2s_rfc7693_vector(bj, ctx):
    """RFC 7693 appendix B: BLAKE2s-256("abc") - checked through a leaf whose bytes start with "abc"... the tree API only
    hashes whole u64 words, so the known-answer here is the empty-row-free vector: 8 zero bytes."""
    import hashlib
    col = np.zeros(1, dtype=np.uint64)
    tree = ctx.merkle_tree_construct([bj.to_device(col)], 1, hasher="blake2s")
    assert bj.to_numpy(tree.leaf_hashes)[0].tobytes() == hashlib.blake2s(bytes(8), digest_size=32).digest()
    assert hashlib.blake2s(b"abc", digest_size=32).hexdigest() == "508c5e8c327c14e2e1a72ba34eeb452f37458b209ed63a294d999b4c86675982"


# ---- setup / witness materialisation (SURVEY 8f rows 1-2) ----
@pytest.mark.parametrize("log_n,n_cols,n_vars", [(4, 3, 10), (6, 5, 40), (8, 7, 3000), (10, 12, 200)])
def test_materialize_columns_and_permutation_polys_match_reference_loops(bj, ctx, log_n, n_cols, n_vars):
    from oracle import setup_oracle as SO
    c = ctx
    rng = np.random.default_rng(log_n * 100 + n_cols)
    n = 1 << log_n
    hint_rows = n - 3
    place = rng.integers(0, n_vars, size=(n_cols, n), dtype=np.uint64)
    place[rng.random((n_cols, n)) < 0.2] = SO.PLACEHOLDER_BIT          # unassigned cells
    values = rng.integers(0, 2**64 - 1, size=n_vars, dtype=np.uint64)
    values[::3] = rng.integers(P, 2**64, size=values[::3].shape, dtype=np.uint64)  # non-canonical words
    hint = np.ascontiguousarray(place[:, :hint_rows])
    got = bj.to_numpy(c.materialize_variables_polynomials_from_dense_hint(bj.to_device(values), bj.to_device(hint), log_n))
    want = SO.materialize_columns([int(v) for v in values], [[int(v) for v in col] for col in hint], n)
    assert got.tolist() == want
    sig = bj.to_numpy(c.create_permutation_polys(bj.to_device(place)))
    want_sig = SO.create_permutation_polys([[int(v) for v in col] for col in place], n)
    assert sig.tolist() == want_sig
    # the sigma columns are a permutation of the identity columns k_c * w^row
    ident = SO.create_permutation_polys([[SO.PLACEHOLDER_BIT] * n for _ in range(n_cols)], n)
    assert sorted(v for col in sig.tolist() for v in col) == sorted(v for col in ident for v in col)


def test_materialize_columns_rejects_out_of_range_hint(bj, ctx):
    c = ctx
    hint = bj.to_device(np.array([[0, 1, 5, 2]], dtype=np.uint64))
    with pytest.raises(bj.BoojumError):
        c.materialize_variables_polynomials_from_dense_hint(bj.to_device(np.arange(4, dtype=np.uint64)), hint, 2)


# ---- error behaviour of the C-ABI: every misuse is a status + message, never an abort (the reference panics instead) ----
def test_c_abi_rejects_misuse_with_status_codes(bj, ctx):
    import ctypes
    import torch
    from era_boojum_b200 import native
    lib, h = native.lib, ctx._h
    dev = "cuda:0"
    t = torch.zeros(64, dtype=torch.int64, device=dev)
    p = ctypes.c_void_p(t.data_ptr())
    INV = native.BJ_ERR_INVALID_ARG
    # NULL pointers / impossible sizes
    assert lib.bj_ntt_natural_to_bitreversed(h, None, 4, 1, 16, 1) == INV
    assert lib.bj_ntt_natural_to_bitreversed(h, p, 33, 1, 1 << 33, 1) == INV           # beyond the 2-adicity of the field
    assert lib.bj_intt_natural_to_natural(h, p, 4, 2, 8, 1) == INV                      # column stride smaller than the column
    assert lib.bj_lde(h, p, 4, p, 4, 1, 1, 0) == INV                                    # in_col_stride < n
    srcs = (ctypes.c_void_p * 1)(t.data_ptr())
    assert lib.bj_merkle_build_poseidon2(h, srcs, 1, 48, 1, 4, p, p) == INV            # leaves not a power of two
    assert lib.bj_merkle_build_poseidon2(h, srcs, 1, 16, 1, 32, p, p) == INV           # cap larger than the tree
    assert lib.bj_merkle_build_blake2s(h, srcs, 1, 16, 3, 4, p, p) == INV              # elems per leaf not a power of two
    al = (ctypes.c_uint64 * 2)(1, 0)
    ci = ctypes.c_uint64(1)
    assert lib.bj_fri_fold(h, p, p, 4, 4, al, ctypes.byref(ci), p, p) == INV           # fold by 16
    assert lib.bj_fri_fold(h, p, p, 2, 3, al, ctypes.byref(ci), p, p) == INV           # fold deeper than the vector
    assert lib.bj_ctx_set_coset_shard(h, 3, 2, 3) == INV                                # rank >= world
    assert lib.bj_ctx_set_coset_shard(h, 0, 16, 3) == INV                               # more shards than cosets
    assert lib.bj_ctx_set_coset_shard(h, 0, 3, 3) == INV                                # world not a power of two
    assert b"coset" in lib.bj_last_error(h) or b"world" in lib.bj_last_error(h)
    sched = (ctypes.c_uint32 * 2)(3, 4)
    out = ctypes.c_void_p()
    tr = ctypes.c_void_p(lib.bj_transcript_new())
    assert lib.bj_do_fri(h, tr, p, p, 6, sched, 2, 1, 4, ctypes.byref(out)) == INV      # fold of 4 in the schedule
    sched = (ctypes.c_uint32 * 2)(3, 3)
    assert lib.bj_do_fri(h, tr, p, p, 6, sched, 2, 1, 4, ctypes.byref(out)) == INV      # final degree would be zero
    assert lib.bj_do_fri_with_hasher(h, tr, p, p, 6, sched, 1, 1, 4, 7, ctypes.byref(out)) == INV   # unknown hasher
    lib.bj_transcript_free(tr)
    # query helpers validate leaf indices on the host before any launch (a bad index from a C / Rust caller is a status, not an
    # out-of-bounds device read)
    idx = (ctypes.c_uint64 * 2)(3, 64)
    hout = (ctypes.c_uint64 * 64)()
    assert lib.bj_query_leaf_elements(h, srcs, 1, 1, 64, idx, 2, hout) == INV          # index 64 of 64 leaves
    assert lib.bj_query_leaf_elements(h, srcs, 1, 1, 65, idx, 2, hout) == 0
    assert lib.bj_merkle_paths(h, p, p, 16, 4, idx, 2, hout) == INV                    # index 64 of 16 leaves
    one = ctypes.c_uint64(0)
    assert lib.bj_selftest_field(h, 0, 1, ctypes.byref(one)) == 0 and one.value == 0   # n == 0: nothing to do, no launch
    # the context stays usable afterwards
    x = O.random_field(rng(1), (1, 16))
    assert np.array_equal(bj.to_numpy(ctx.fft_natural_to_bitreversed(bj.to_device(x), 1)), O.ntt_n2b(x, 1))


def test_entry_points_run_on_the_device_of_their_context(bj):
    """A context stays bound to its device whatever the caller's current device is (two contexts on two GPUs in one thread
    when the box has them; otherwise the current device is moved away with a second context on the same GPU), and no entry
    point leaves the caller's current device changed."""
    import torch
    n_dev = torch.cuda.device_count()
    other = 1 if n_dev > 1 else 0
    x = O.random_field(rng(9), (2, 1 << 10))
    want = O.ntt_n2b(x, 7)
    torch.cuda.set_device(0)
    c0 = bj.Context(0)
    torch.cuda.set_device(other)
    c1 = bj.Context(other)
    assert torch.cuda.current_device() == other
    d0, d1 = bj.to_device(x, "cuda:0"), bj.to_device(x, "cuda:%d" % other)
    c0.fft_natural_to_bitreversed(d0, 7)                  # current device is `other`, the context lives on 0
    assert torch.cuda.current_device() == other
    torch.cuda.set_device(0)
    c1.fft_natural_to_bitreversed(d1, 7)                  # and the other way round
    tree = c1.merkle_tree_construct([d1[0], d1[1]], 4)
    assert torch.cuda.current_device() == 0
    c0.synchronize(), c1.synchronize()
    assert np.array_equal(bj.to_numpy(d0), want) and np.array_equal(bj.to_numpy(d1), want)
    lh, _, cap = O.merkle_tree([want[0], want[1]], 4)
    assert np.array_equal(tree.get_cap(), cap)
    c0.close(), c1.close()
    torch.cuda.set_device(0)


@pytest.mark.parametrize("n_cols,log_leaves,cap,epl", [(1, 3, 1, 1), (8, 5, 4, 1), (17, 6, 8, 1), (18, 4, 2, 1), (93, 7, 16, 1), (2, 6, 4, 8), (34, 3, 8, 1)])
def test_merkle_keccak256_matches_oracle(bj, ctx, n_cols, log_leaves, cap, epl):
    """impl TreeHasher for sha3::Keccak256 (src/cs/oracle/mod.rs:247-313): leaves over 1, <17, =17, >17 and a multiple of
    17 lanes (the rate is 17 u64), chunked leaves, caps from 1 to the number of leaves."""
    n = 1 << log_leaves
    cols = [O.random_field(rng(100 + c), n * epl) for c in range(n_cols)]
    if n_cols > 2:
        cols[1][:] = np.uint64(0xFFFFFFFFFFFFFFFF)          # non-canonical input: hashed as its reduced value
    tree = ctx.merkle_tree_construct([bj.to_device(c) for c in cols], cap, elems_per_leaf=epl, hasher="keccak256")
    leaves = [replay.keccak_leaf_hash([int(v) for c in cols for v in c[i * epl:(i + 1) * epl]]) for i in range(n)]
    assert np.array_equal(bj.to_numpy(tree.leaf_hashes), np.array(leaves, dtype=np.uint64))
    level = leaves
    while len(level) > cap:
        level = [replay.keccak_node_hash(level[2 * i], level[2 * i + 1]) for i in range(len(level) // 2)]
    assert np.array_equal(tree.get_cap(), np.array(level, dtype=np.uint64))
