"""Split domain shards: more ranks than LDE cosets (bj_ctx_set_domain_shard with world > L).  Every coset is cut into
B = world / L row blocks; the units u = j * B + p are dealt out round robin (rank r holds u = r mod world, [local unit][n / B]).
Each entry point is compared bit for bit with the unsharded result (or the CPU oracle) sliced the same way, and the native
driver, run with thread ranks over the local transport, must return the single-GPU proof on every rank."""
import ctypes
import json
import threading

import numpy as np
import pytest

from oracle import oracle as O
from oracle import verifier as OV

pytestmark = pytest.mark.gpu

P = O.P
INV = -1          # BJ_ERR_INVALID_ARG
UNSUPPORTED = -5  # BJ_ERR_UNSUPPORTED


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


@pytest.fixture
def ctx(bj):
    c = bj.Context(0)
    yield c
    c.synchronize()
    c.close()


def _field(seed, shape):
    """canonical values, about one in seven replaced by a non-canonical one in [p, 2^64)"""
    r = np.random.default_rng(seed)
    a = O.random_field(r, shape)
    mask = r.random(shape) < 1 / 7
    a[mask] = r.integers(P, 2**64, size=int(mask.sum()), dtype=np.uint64)
    return a


def _units(flat, n_units):
    """[..., D * n] or [..., D, n] -> [..., units, n * D / units]"""
    a = np.asarray(flat)
    lead = a.shape[:-2] if a.ndim >= 3 else a.shape[:-1]
    return a.reshape(*lead, n_units, -1)


def _bitrev(x, bits):
    return int(format(x, "0%db" % bits)[::-1], 2) if bits else 0


# ------------------------------------------------------------------------------------------ 1. LDE onto row blocks -----
@pytest.mark.parametrize("from_mono", [False, True])
@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("lde,world", [(2, 4), (2, 8), (2, 16), (4, 8)])
def test_split_lde_equals_unit_slices(bj, ctx, lde, world, small, from_mono):
    B = world // lde
    log_n = (B.bit_length()) if small else 12            # small: n / B == 2
    n, cols, log_l = 1 << log_n, 3, lde.bit_length() - 1
    a = _field(100 * world + 10 * lde + small, (cols, n))
    want = _units(O.lde(a, log_l, from_monomials=from_mono), lde * B)
    for rank in range(world):
        ctx.set_domain_shard(rank, world, lde)
        out = ctx.transform_raw_storages_to_lde(bj.to_device(a), lde, from_monomials=from_mono)
        assert tuple(out.shape) == (cols, lde * B // world, n // B)
        got = bj.to_numpy(out)
        assert (got < P).all()
        assert np.array_equal(got, want[:, rank::world]), rank


def test_split_lde_wider_domain(bj, ctx):
    """a shard declared for L = 2 at world 4 (B = 2), asked for 8 cosets (the quotient's wider domain): 16 units, 4 per rank"""
    log_n, cols = 10, 2
    a = _field(7, (cols, 1 << log_n))
    want = _units(O.lde(a, 3), 16)
    for rank in range(4):
        ctx.set_domain_shard(rank, 4, 2)
        out = ctx.transform_raw_storages_to_lde(bj.to_device(a), 8)
        assert tuple(out.shape) == (cols, 4, (1 << log_n) // 2)
        assert np.array_equal(bj.to_numpy(out), want[:, rank::4])


def test_domain_shard_without_split_is_the_coset_shard(bj, ctx):
    """world <= L: set_domain_shard gives exactly set_coset_shard's cosets"""
    a = _field(11, (2, 1 << 9))
    want = O.lde(a, 3)
    for rank in range(4):
        ctx.set_domain_shard(rank, 4, 8)
        assert np.array_equal(bj.to_numpy(ctx.transform_raw_storages_to_lde(bj.to_device(a), 8)), want[:, rank::4])


# ------------------------------------------------------------------------------------------ 2. z(omega x) columns -----
@pytest.mark.parametrize("lde,world,log_n", [(2, 4, 10), (2, 8, 9), (4, 16, 8), (2, 16, 4)])
def test_next_row_lde_is_the_in_coset_shift(bj, ctx, lde, world, log_n):
    """bj_lde_next_row on a split shard == the unsharded LDE permuted by bitrev(bitrev(i) + 1) inside each coset"""
    n, log_l, B = 1 << log_n, lde.bit_length() - 1, world // lde
    z = _field(3 * world + log_n, (2, n))
    full = O.lde(z, log_l)
    nxt = [_bitrev((_bitrev(i, log_n) + 1) % n, log_n) for i in range(n)]
    want = _units(full[:, :, nxt], lde * B)
    for rank in range(world):
        ctx.set_domain_shard(rank, world, lde)
        out = ctx.transform_raw_storages_to_lde(bj.to_device(z), lde, next_row=True)
        assert np.array_equal(bj.to_numpy(out), want[:, rank::world]), rank


# ------------------------------------------------------------------------------------------ 3. openings -----
@pytest.mark.parametrize("lde,world", [(2, 4), (2, 16), (4, 8)])
def test_barycentric_contributions_sum_to_the_value(bj, ctx, lde, world):
    log_n, cols, B = 10, 5, world // lde
    a = _field(50 + world, (cols, 1 << log_n))
    at = (0x1234567887654321 % P, 0x0FEDCBA987654321 % P)
    full = ctx.transform_raw_storages_to_lde(bj.to_device(a), lde)
    want = ctx.barycentric_evaluate([full[c].reshape(-1) for c in range(cols)], log_n, at)
    contrib = []
    for rank in range(world):
        ctx.set_domain_shard(rank, world, lde)
        loc = ctx.transform_raw_storages_to_lde(bj.to_device(a), lde)
        contrib.append(ctx.barycentric_evaluate([loc[c].reshape(-1) for c in range(cols)], log_n, at))
    ctx.set_coset_shard(0, 1, lde)
    for g in range(lde):                                   # every coset group gives the value on its own
        got = []
        for c in range(cols):
            s0 = s1 = 0
            for p in range(B):
                s0, s1 = O.add(s0, contrib[g * B + p][c][0]), O.add(s1, contrib[g * B + p][c][1])
            got.append((s0, s1))
        assert got == want, g
    assert contrib[0] != want                              # one block alone is only a part


# ------------------------------------------------------------------------------------------ 4. FRI fold and DEEP -----
@pytest.mark.parametrize("lde,world,log_fold", [(2, 4, 3), (2, 16, 2), (4, 8, 1)])
def test_fri_fold_on_units(bj, ctx, lde, world, log_fold):
    log_m = 12
    c0, c1 = (bj.to_device(_field(s, 1 << log_m)) for s in (1, 2))
    alpha, kappa = (123456789, 987654321), O.inv(7)
    o0, o1, k_ref = ctx.fri_fold(c0, c1, log_fold, alpha, kappa)
    units = world                                          # L * B
    w0, w1 = _units(bj.to_numpy(o0), units), _units(bj.to_numpy(o1), units)
    u0, u1 = _units(bj.to_numpy(c0), units), _units(bj.to_numpy(c1), units)
    for rank in range(world):
        ctx.set_domain_shard(rank, world, lde)
        l0, l1 = (bj.to_device(np.ascontiguousarray(u[rank::world]).reshape(-1)) for u in (u0, u1))
        g0, g1, k = ctx.fri_fold(l0, l1, log_fold, alpha, kappa)
        assert k == k_ref
        assert np.array_equal(bj.to_numpy(g0), w0[rank::world].reshape(-1))
        assert np.array_equal(bj.to_numpy(g1), w1[rank::world].reshape(-1))


@pytest.mark.parametrize("lde,world", [(2, 8), (4, 16)])
def test_deep_quotient_on_units(bj, ctx, lde, world):
    import torch
    log_n, n_src = 9, 3
    units = world
    srcs = [bj.to_device(_field(10 + i, lde << log_n)) for i in range(2 * n_src)]
    sources = [(srcs[0], None), (srcs[1], srcs[2]), (srcs[3], srcs[4])]
    vals = [(5, 6), (7, 8), (9, 10)]
    chs = [(11, 12), (13, 14), (15, 16)]
    at = (0x1111222233334444, 0x5555666677778888)
    z = lambda m: torch.zeros(m, dtype=torch.int64, device="cuda:0")
    a0, a1 = ctx.quotening_operation_in_extension(z(lde << log_n), z(lde << log_n), sources, vals, at, chs)
    w0, w1 = _units(bj.to_numpy(a0), units), _units(bj.to_numpy(a1), units)
    for rank in range(world):
        ctx.set_domain_shard(rank, world, lde)
        loc = lambda t: None if t is None else bj.to_device(np.ascontiguousarray(_units(bj.to_numpy(t), units)[rank::world]).reshape(-1))
        ls = [(loc(s0), loc(s1)) for s0, s1 in sources]
        m = (lde << log_n) // world
        g0, g1 = ctx.quotening_operation_in_extension(z(m), z(m), ls, vals, at, chs)
        assert np.array_equal(bj.to_numpy(g0), w0[rank::world].reshape(-1))
        assert np.array_equal(bj.to_numpy(g1), w1[rank::world].reshape(-1))


# ------------------------------------------------------------------------------------------ 5. end to end -----
def _prove_native_sharded_threads(bj, world, lde, cap, cfg, circuit, Q):
    """the library's sharded driver: `world` ranks as threads on one GPU over the local transport, every rank on the same
    (shared, read-only) circuit tensors; returns every rank's (cap, proof)"""
    group = bj.Comm.local_group(world)
    out, errs = [None] * world, []

    def run(rank):
        try:
            ctx = bj.Context(0)
            comm = bj.Comm.local(ctx, group, rank, world, lde)
            nat = ctx.native_setup(circuit["sigmas"], circuit["constants"], circuit["gates"], Q, cfg, lookup=circuit["lookup"],
                                   public_inputs=circuit["public_inputs"])
            m = circuit["lookup"]["multiplicities"] if circuit["lookup"] else None
            proof = nat.prove(circuit["variables"], m)
            out[rank] = (nat.get_cap(), proof)
            ctx.synchronize()
            nat.close()
            comm.close()
            ctx.close()
        except BaseException as e:
            errs.append(e)

    ts = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(world)]
    [t.start() for t in ts]
    [t.join(timeout=900) for t in ts]
    if errs:
        raise errs[0]
    assert all(o is not None for o in out), "a rank did not finish"
    bj.Comm.destroy_local_group(group)
    return out


def _check_sharded_equals_single(bj, world, lde, cap, hasher, transcript, circuit, Q):
    from era_boojum_b200 import prover
    import torch
    torch.cuda.synchronize()
    cfg = prover.ProofConfig(fri_lde_factor=lde, merkle_tree_cap_size=cap, security_level=100, hasher=hasher, transcript=transcript)
    ctx = bj.Context(0)
    nat = ctx.native_setup(circuit["sigmas"], circuit["constants"], circuit["gates"], Q, cfg, lookup=circuit["lookup"],
                           public_inputs=circuit["public_inputs"])
    ref = nat.prove(circuit["variables"], circuit["lookup"]["multiplicities"] if circuit["lookup"] else None)
    assert OV.verify(nat.vk(), ref)
    ref_cap = nat.get_cap()
    nat.close()
    ctx.synchronize()
    ctx.close()
    res = _prove_native_sharded_threads(bj, world, lde, cap, cfg, circuit, Q)
    want = json.dumps(ref, sort_keys=True)
    for rank, (cap_r, proof) in enumerate(res):
        assert np.array_equal(cap_r, ref_cap), rank
        assert json.dumps(proof, sort_keys=True) == want, rank


def _synthetic(bj, log_n, V, lookup, pis):
    from era_boojum_b200 import synthetic
    ctx = bj.Context.on_current_stream(0)
    gen = synthetic.generate(ctx, log_n, V, seed=3, lookup=lookup)
    variables, sigmas, constants, gates, Q = gen[:5]
    c = {"variables": variables.contiguous(), "sigmas": sigmas.contiguous(), "constants": constants.contiguous(), "gates": gates,
         "lookup": gen[5] if lookup else None, "public_inputs": pis}
    ctx.synchronize()
    ctx.close()
    return c, Q


@pytest.mark.parametrize("world,log_n,V,lde,cap,lookup,hasher,transcript,pis", [
    (4, 10, 60, 2, 16, True, "poseidon2", "poseidon2", [(1, 3), (5, 3)]),
    (8, 10, 60, 2, 16, False, "poseidon2", "poseidon", []),
    (8, 9, 60, 4, 16, True, "blake2s", "blake2s", [(2, 7)]),
    (16, 10, 20, 4, 16, False, "keccak256", "keccak256", [])])
def test_split_sharded_prover_equals_single_gpu(bj, world, log_n, V, lde, cap, lookup, hasher, transcript, pis):
    """L = 2 (quotient degree 4 > L) at world 4 and 8, L = 4 at world 8 and 16; with and without lookups and public inputs;
    each hasher / transcript pair once"""
    circuit, Q = _synthetic(bj, log_n, V, lookup, pis)
    assert world > lde
    _check_sharded_equals_single(bj, world, lde, cap, hasher, transcript, circuit, Q)


@pytest.fixture(scope="module")
def production(bj):
    from era_boojum_b200 import synthetic
    ctx = bj.Context.on_current_stream(0)
    c = synthetic.generate_production_shaped(ctx, 11, seed=5)
    ctx.synchronize()
    ctx.close()
    return c


@pytest.mark.parametrize("world", [4, 8, 16])
def test_production_shaped_split_sharded(bj, production, world):
    """the production shape (155 columns, Q = 8 over L = 2, cap 32) spread over 4, 8 and 16 ranks"""
    _check_sharded_equals_single(bj, world, 2, 32, "poseidon2", "poseidon2", production, 8)


# ------------------------------------------------------------------------------------------ 6. misuse -----
def test_domain_shard_limits(bj, ctx):
    lib = bj.native.lib
    h = ctx._h
    assert lib.bj_ctx_set_domain_shard(h, 0, 32, 1) == INV        # more than 8 row blocks per coset
    assert b"8 * the LDE factor" in lib.bj_last_error(h)
    assert lib.bj_ctx_set_domain_shard(h, 0, 12, 1) == INV        # not a power of two
    assert lib.bj_ctx_set_domain_shard(h, 4, 4, 1) == INV         # rank >= world
    assert lib.bj_ctx_set_domain_shard(h, 3, 16, 1) == 0
    assert lib.bj_ctx_set_coset_shard(h, 0, 16, 3) == INV         # the coset shard keeps its limit
    assert lib.bj_ctx_set_coset_shard(h, 0, 1, 1) == 0


def _setup_error(bj, world, lde, cap, log_n):
    """bj_setup_create on rank 0 of a local communicator: (status, message, kernels launched by the call)"""
    from era_boojum_b200 import prover
    circuit, Q = _synthetic(bj, log_n, 20, False, [])
    group = bj.Comm.local_group(world)
    c = bj.Context(0)
    comm = bj.Comm.local(c, group, 0, world, lde)
    cfg = prover.ProofConfig(fri_lde_factor=lde, merkle_tree_cap_size=cap, security_level=100)
    before = c.launch_count()
    try:
        with pytest.raises(bj.BoojumError) as e:
            c.native_setup(circuit["sigmas"], circuit["constants"], circuit["gates"], Q, cfg)
        return e.value, c.launch_count() - before
    finally:
        comm.close()
        c.close()
        bj.Comm.destroy_local_group(group)


def test_setup_refuses_cap_smaller_than_world(bj):
    err, launched = _setup_error(bj, 16, 2, 8, 10)
    assert err.status == INV and "cap_size >= max(LDE factor, world)" in str(err)
    assert launched == 0


def test_setup_refuses_one_row_blocks(bj):
    err, launched = _setup_error(bj, 16, 2, 16, 3)
    assert err.status == INV and "at least 2 rows" in str(err)
    assert launched == 0


def test_fold_refuses_units_shorter_than_the_fold(bj, ctx):
    """world 8 over L = 2: units of a 2^4 codeword hold 2 elements, a fold by 4 would cross them"""
    import torch
    ctx.set_domain_shard(0, 8, 2)
    c0, c1, o0, o1 = (torch.zeros(2, dtype=torch.int64, device="cuda:0") for _ in range(4))
    al, ci = (ctypes.c_uint64 * 2)(1, 2), ctypes.c_uint64(3)
    before = ctx.launch_count()
    st = bj.native.lib.bj_fri_fold(ctx._h, ctx._ptr(c0), ctx._ptr(c1), 4, 2, al, ctypes.byref(ci), ctx._ptr(o0), ctx._ptr(o1))
    assert st == INV and b"cross units" in bj.native.lib.bj_last_error(ctx._h)
    assert ctx.launch_count() == before


def test_copy_permutation_quotient_needs_z_next_on_split_shard(bj, ctx):
    import torch
    ctx.set_domain_shard(1, 4, 2)
    t, q0, q1 = (torch.zeros(1 << 10, dtype=torch.int64, device="cuda:0") for _ in range(3))
    args = ([t], [t], (t, t), [], (1, 2), (3, 4), [(1, 0), (2, 0)], 9, 1, 1, 4, q0, q1)
    before = ctx.launch_count()
    with pytest.raises(bj.BoojumError) as e:
        ctx.quotient_copy_permutation(*args)
    assert e.value.status == UNSUPPORTED and "bj_quotient_copy_permutation_with_z_next" in str(e.value)
    assert ctx.launch_count() == before
    ctx.set_domain_shard(1, 2, 2)                                 # a whole coset: the in-coset shift is still there
    ctx.quotient_copy_permutation(*args)
    ctx.synchronize()
