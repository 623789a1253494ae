"""Proving under a device-memory limit (bj_ctx_set_memory_limit).  A limit between the compact and the resident plan of
bj_proof_memory_plan makes bj_setup_create choose the compact plan: cosets [Q, L) of the setup, witness and stage-2 columns are
dropped after their trees are built and recomputed for DEEP and the query answers.  The proof must not move: it is compared bit
for bit with the unlimited proof and with the oracle's CPU prover, the verifier must accept it, and the context's pool must
stay under the limit.  Limits below the compact plan, and limits on contexts where only the resident plan applies (quotient
degree >= LDE factor, sharded contexts), are refused with BJ_ERR_OOM before any kernel runs."""
import ctypes
import json
import threading

import numpy as np
import pytest

from oracle import oracle as O
from oracle import verifier as OV

pytestmark = pytest.mark.gpu

INV = -1          # BJ_ERR_INVALID_ARG
OOM = -4          # BJ_ERR_OOM
UNSUPPORTED = -5  # BJ_ERR_UNSUPPORTED


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


def _circuit(bj, log_n, V, Q, lookup):
    """the oracle's SHA-shaped circuit; Q = 2 drops the gates (their degree needs Q = 4) and proves the copy permutation and
    lookup argument alone"""
    from era_boojum_b200 import synthetic
    from oracle import circuits
    c = circuits.sha_shaped(log_n, V, seed=200 + log_n, lookup=lookup)
    gates, oracle_gates = synthetic.sha_shaped_gates(V), c["gates"]
    if Q == 2:
        gates, oracle_gates = [], []
    return c, gates, oracle_gates


def _setup(bj, ctx, c, gates, Q, cfg, pis):
    lk = None
    if c["lookup"]:
        lk = dict(c["lookup"], tables=bj.to_device(c["lookup"]["tables"]), multiplicities=bj.to_device(c["lookup"]["multiplicities"]))
    dev = dict(sigmas=bj.to_device(c["sigmas"]), constants=bj.to_device(c["constants"]), variables=bj.to_device(c["variables"]), lk=lk)
    nat = ctx.native_setup(dev["sigmas"], dev["constants"], gates, Q, cfg, lookup=lk, public_inputs=list(pis))
    return nat, dev


def _num_queries(bj, log_n, cfg):
    new_pow, nq, sl, fd = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    sched = (ctypes.c_uint32 * 32)()
    assert bj.native.lib.bj_compute_fri_schedule(cfg.security_level, cfg.merkle_tree_cap_size, cfg.pow_bits, cfg.fri_lde_factor.bit_length() - 1,
                                                 log_n, ctypes.byref(new_pow), ctypes.byref(nq), sched, ctypes.byref(sl), ctypes.byref(fd)) == 0
    return nq.value


def _check_high_water(bj, ctx, nat, log_n, cfg):
    """the pool's high-water mark over setup + prove on a fresh context is the planned pool peak.  The one allowance: the
    compact plan's gather of recomputed query rows is planned for every query, and only the queries whose leaf lies in a
    dropped coset use it."""
    mp = nat.memory_plan()
    high = ctx.memory_high_water()
    slack = 8 * _num_queries(bj, log_n, cfg) * mp["chunk"]
    assert mp["pool"] - slack <= high <= mp["pool"], (high, mp)
    return high, mp


def _plan(bj, c, Q, cfg):
    lk = dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"]) if c["lookup"] else None
    return bj.proof_memory_plan(c["sigmas"].shape[1].bit_length() - 1, c["sigmas"].shape[0], c["constants"].shape[0], Q, cfg, lookup=lk)


@pytest.mark.parametrize("log_n,V,L,Q,lookup,pis,hasher,transcript", [
    (9, 20, 8, 4, False, (), "poseidon2", "poseidon2"),
    (10, 20, 8, 4, True, ((1, 3), (5, 3)), "blake2s", "blake2s"),
    (11, 40, 8, 4, True, ((2, 100),), "poseidon2", "poseidon"),
    (12, 20, 8, 4, False, ((0, 9),), "keccak256", "keccak256"),
    (9, 20, 4, 2, True, ((0, 1), (19, 511)), "poseidon2", "poseidon2"),
    (10, 20, 4, 2, False, (), "blake2s", "blake2s"),
    (12, 20, 4, 2, True, ((3, 5),), "poseidon2", "poseidon")])
def test_compact_plan_proves_the_same_proof_under_the_limit(bj, log_n, V, L, Q, lookup, pis, hasher, transcript):
    from era_boojum_b200 import prover
    from oracle import prover as OP
    c, gates, oracle_gates = _circuit(bj, log_n, V, Q, lookup)
    cfg = prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=16 if L == 8 else 8, security_level=100, hasher=hasher,
                             transcript=transcript)
    plan = _plan(bj, c, Q, cfg)
    assert plan["compact"] is not None and plan["compact"] < plan["resident"]
    limit = (plan["compact"] + plan["resident"]) // 2

    ctx = bj.Context(0)
    nat, dev = _setup(bj, ctx, c, gates, Q, cfg, pis)
    assert not nat.compact
    m = dev["lk"]["multiplicities"] if lookup else None
    want = nat.prove(dev["variables"], m)
    want_cap = nat.get_cap()
    high_resident, _ = _check_high_water(bj, ctx, nat, log_n, cfg)
    nat.close()
    ctx.synchronize()
    ctx.close()

    ctx = bj.Context(0)
    ctx.set_memory_limit(limit)
    nat, dev = _setup(bj, ctx, c, gates, Q, cfg, pis)
    assert nat.compact
    got = nat.prove(dev["variables"], dev["lk"]["multiplicities"] if lookup else None)
    high, mp = _check_high_water(bj, ctx, nat, log_n, cfg)
    assert mp["pool"] + mp["outside_pool"] <= limit
    # the compact plan keeps less on the device than the resident one did for the same proof
    assert high < high_resident
    assert np.array_equal(nat.get_cap(), want_cap)
    assert json.dumps(got, sort_keys=True) == json.dumps(want, sort_keys=True)
    assert OV.verify(nat.vk(), got)
    nat.close()
    ctx.synchronize()
    ctx.close()

    if log_n <= 10:  # the oracle's CPU prover (Python integers) on the smaller shapes
        ref, ref_cap = OP.prove(c["variables"], c["sigmas"], c["constants"], oracle_gates, Q, L, cfg.merkle_tree_cap_size,
                                lookup=c["lookup"], public_inputs=pis, hasher=hasher, transcript=transcript)
        assert np.array_equal(want_cap, ref_cap)
        assert json.dumps(got, sort_keys=True) == json.dumps(ref, sort_keys=True)


def test_limit_below_the_compact_plan_is_refused(bj):
    from era_boojum_b200 import prover
    c, gates, _ = _circuit(bj, 10, 20, 4, True)
    cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)
    plan = _plan(bj, c, 4, cfg)
    ctx = bj.Context(0)
    ctx.set_memory_limit(plan["compact"] - 1)
    before = ctx.launch_count()
    with pytest.raises(bj.BoojumError) as e:
        _setup(bj, ctx, c, gates, 4, cfg, ())
    assert e.value.status == OOM
    assert str(plan["resident"]) in str(e.value) and str(plan["compact"]) in str(e.value)
    assert ctx.launch_count() == before
    ctx.close()


def test_prove_refuses_a_limit_lowered_below_the_plan(bj):
    from era_boojum_b200 import prover
    c, gates, _ = _circuit(bj, 9, 20, 4, False)
    cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)
    plan = _plan(bj, c, 4, cfg)
    ctx = bj.Context(0)
    nat, dev = _setup(bj, ctx, c, gates, 4, cfg, ())
    assert not nat.compact
    ctx.set_memory_limit(plan["resident"] - 1)
    ctx.synchronize()
    before = ctx.launch_count()
    with pytest.raises(bj.BoojumError) as e:
        nat.prove(dev["variables"])
    assert e.value.status == OOM and str(plan["resident"]) in str(e.value)
    assert ctx.launch_count() == before
    nat.close()
    ctx.close()


def test_quotient_degree_at_least_the_lde_factor_keeps_resident(bj):
    """L = 4, Q = 4: no compact plan; a limit below the resident plan refuses, one above it proves resident"""
    from era_boojum_b200 import prover
    c, gates, _ = _circuit(bj, 9, 20, 4, True)
    cfg = prover.ProofConfig(fri_lde_factor=4, merkle_tree_cap_size=8, security_level=100)
    plan = _plan(bj, c, 4, cfg)
    assert plan["compact"] is None
    ctx = bj.Context(0)
    ctx.set_memory_limit(plan["resident"] - 1)
    before = ctx.launch_count()
    with pytest.raises(bj.BoojumError) as e:
        _setup(bj, ctx, c, gates, 4, cfg, ())
    assert e.value.status == OOM and "no compact plan" in str(e.value) and str(plan["resident"]) in str(e.value)
    assert ctx.launch_count() == before
    ctx.set_memory_limit(plan["resident"])
    nat, dev = _setup(bj, ctx, c, gates, 4, cfg, ())
    assert not nat.compact
    proof = nat.prove(dev["variables"], dev["lk"]["multiplicities"])
    _check_high_water(bj, ctx, nat, 9, cfg)
    assert OV.verify(nat.vk(), proof)
    nat.close()
    ctx.close()


def test_sharded_context_keeps_resident(bj):
    """a limit on rank 0 of a 2-rank context: the per-GPU resident plan is the only one; below it the setup is refused"""
    from era_boojum_b200 import prover
    c, gates, _ = _circuit(bj, 10, 20, 4, False)
    cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)
    single = _plan(bj, c, 4, cfg)
    sharded = bj.proof_memory_plan(10, 20, c["constants"].shape[0], 4, cfg, world=2)
    assert sharded["compact"] is None
    group = bj.Comm.local_group(2)
    ctx = bj.Context(0)
    comm = bj.Comm.local(ctx, group, 0, 2, 8)
    ctx.set_memory_limit(min(single["compact"], sharded["resident"] - 1))
    before = ctx.launch_count()
    result = []

    def run():  # the other rank never joins: were the refusal to come after the first collective, this would block
        try:
            _setup(bj, ctx, c, gates, 4, cfg, ())
            result.append(None)
        except bj.BoojumError as e:
            result.append(e)

    t = threading.Thread(target=run, daemon=True)
    t.start()
    t.join(timeout=120)
    assert not t.is_alive(), "bj_setup_create did not refuse before its first collective"
    try:
        e = result[0]
        assert e is not None, "bj_setup_create accepted a limit below the sharded resident plan"
        assert e.status == OOM and "no compact plan" in str(e) and str(sharded["resident"]) in str(e)
        assert ctx.launch_count() == before
    finally:
        comm.close()
        ctx.close()
        bj.Comm.destroy_local_group(group)


# ---------------------------------------------------------------- the two entry points the compact plan is built on -----
def _field(seed, shape):
    """canonical values, about one in seven replaced by a non-canonical one in [p, 2^64)"""
    r = np.random.default_rng(seed)
    a = O.random_field(r, shape)
    mask = r.random(shape) < 1 / 7
    a[mask] = r.integers(O.P, 2**64, size=int(mask.sum()), dtype=np.uint64)
    return a


@pytest.mark.parametrize("from_mono", [False, True])
@pytest.mark.parametrize("log_n,L,j0,j1", [(10, 8, 0, 8), (10, 8, 3, 6), (10, 8, 7, 8), (3, 4, 1, 3), (17, 2, 1, 2)])
def test_lde_cosets_equals_the_slots_of_the_full_lde(bj, log_n, L, j0, j1, from_mono):
    ctx = bj.Context(0)
    cols = 5
    d = bj.to_device(_field(log_n + j0, (cols, 1 << log_n)))
    if from_mono:
        d = ctx.ifft_natural_to_natural(d.clone())
    full = bj.to_numpy(ctx.transform_raw_storages_to_lde(d, L, from_monomials=from_mono))
    out = ctx._torch.zeros((cols, j1 - j0, 1 << log_n), dtype=ctx._torch.int64, device="cuda:0")
    ctx._check(bj.native.lib.bj_lde_cosets(ctx._h, ctx._ptr(d), 1 << log_n, ctx._ptr(out), log_n, L.bit_length() - 1, j0, j1, cols,
                                           int(from_mono)))
    assert np.array_equal(bj.to_numpy(out), full[:, j0:j1])
    ctx.close()


def _deep_args(sources, vals, chs, at):
    n_src = len(sources)
    p0 = (ctypes.c_void_p * n_src)(*[s[0].data_ptr() for s in sources])
    p1 = (ctypes.c_void_p * n_src)(*[(s[1].data_ptr() if s[1] is not None else None) for s in sources])
    v = (ctypes.c_uint64 * (2 * n_src))(*[x for p in vals for x in p])
    ch = (ctypes.c_uint64 * (2 * n_src))(*[x for p in chs for x in p])
    return p0, p1, n_src, v, ch, (ctypes.c_uint64 * 2)(*at)


def test_deep_quotient_range_pieces_equal_the_whole_domain(bj):
    """the domain cut at points that are not coset boundaries: every piece accumulates exactly the whole-domain result"""
    import torch
    ctx = bj.Context(0)
    L, log_n = 4, 9
    N = L << log_n
    srcs = [bj.to_device(_field(30 + i, N)) for i in range(5)]
    sources = [(srcs[0], None), (srcs[1], srcs[2]), (srcs[3], srcs[4])]
    vals, chs = [(5, 6), (7, 8), (9, 10)], [(11, 12), (13, 14), (15, 16)]
    at = (0x1111222233334444, 0x5555666677778888)
    z = lambda m: torch.zeros(m, dtype=torch.int64, device="cuda:0")
    w0, w1 = ctx.quotening_operation_in_extension(z(N), z(N), sources, vals, at, chs)
    lib = bj.native.lib
    for first, count in [(0, 700), (700, 800), (1500, N - 1500), (0, N)]:
        piece = [(s0[first:first + count].contiguous(), None if s1 is None else s1[first:first + count].contiguous()) for s0, s1 in sources]
        a0, a1 = z(count), z(count)
        ctx._check(lib.bj_deep_quotient_range(ctx._h, *_deep_args(piece, vals, chs, at), log_n + 2, first, count, ctx._ptr(a0), ctx._ptr(a1)))
        assert np.array_equal(bj.to_numpy(a0), bj.to_numpy(w0)[first:first + count]), first
        assert np.array_equal(bj.to_numpy(a1), bj.to_numpy(w1)[first:first + count]), first
    before = ctx.launch_count()
    a0 = z(N)
    assert lib.bj_deep_quotient_range(ctx._h, *_deep_args(sources, vals, chs, at), log_n + 2, 1, N, ctx._ptr(a0), ctx._ptr(a0)) == INV
    ctx.set_coset_shard(0, 2, L)
    assert lib.bj_deep_quotient_range(ctx._h, *_deep_args(sources, vals, chs, at), log_n + 2, 0, N // 2, ctx._ptr(a0), ctx._ptr(a0)) == UNSUPPORTED
    out = z(N)
    assert lib.bj_lde_cosets(ctx._h, ctx._ptr(srcs[0]), 1 << log_n, ctx._ptr(out), log_n, 2, 0, 1, 1, 0) == UNSUPPORTED
    assert ctx.launch_count() == before
    ctx.close()
