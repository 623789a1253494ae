"""bj_proof_memory_plan_recompute_sharded (no GPU): the recompute plan on each rank of a sharded context, counted from the
circuit's shapes.  Every rank keeps no coset of the setup, witness and stage-2 columns and works on its own units u = rank
(mod world): whole cosets on a coset shard (world <= L), row blocks of nb = n / B rows on a split shard (world = L * B).  The
plan is checked against the driver's pool allocations on one rank, listed here one by one in the order prover.cu makes them,
against the single-GPU recompute plan at world 1, and against the sharded resident and streamed plans."""
import ctypes

import pytest

GB = 10**9
INVALID_ARG = -1

# the production shape (155 columns, 8 constants, 8 lookups of width 3, Q = 8 over L = 2, cap 32), the bench shape (60 columns
# and the 32 its 8 lookups of width 4 read, 7 constants, Q = 4 over L = 8, cap 16) and a Q = L shape
SHAPES = {"production": (155, 8, 8, 2, 32, (3, 8)), "bench": (92, 7, 4, 8, 16, (4, 8)), "q_equals_l": (92, 7, 4, 4, 16, (4, 8))}


@pytest.fixture(scope="module")
def bj():
    import era_boojum_b200 as m
    return m


def _cfg(L, cap):
    from era_boojum_b200 import prover
    return prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100)


def _schedule(bj, log_n, L, cap):
    lib = bj.native.lib
    new_pow, nq, sl, fd = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    sched = (ctypes.c_uint32 * 32)()
    assert lib.bj_compute_fri_schedule(100, cap, 0, L.bit_length() - 1, log_n, ctypes.byref(new_pow), ctypes.byref(nq), sched,
                                       ctypes.byref(sl), ctypes.byref(fd)) == 0
    return list(sched[:sl.value]), nq.value


def _recompute_sharded_allocations(bj, log_n, V, C, Q, L, cap, lookup, world, chunk=2):
    """the recompute driver's pool allocations on one rank of `world`, in order: ("+" | "-", u64 count, what)"""
    n = 1 << log_n
    split = max(0, world.bit_length() - L.bit_length())   # log2(B), B = world / L row blocks per coset when world > L
    nb = n >> split
    T = lookup[0] + 1 if lookup else 0
    S, W = V + C + T, V + (1 if lookup else 0)
    n_s2 = 2 + 2 * ((V + Q - 1) // Q - 1) + (2 * (lookup[1] + 1) if lookup else 0)
    nL, nQ = n * L // world, n * Q               # nL: this rank's part of a committed column
    capl = cap // world
    sharded = world > 1
    ev = []
    a = lambda cnt, what: ev.append(("+", cnt, what))
    f = lambda cnt, what: ev.append(("-", cnt, what))

    def tree(what):
        a(4 * nL, what + " leaf hashes")
        a(4 * (nL - capl), what + " nodes")

    def tree_by_unit(what, cols):
        a(4 * nL, what + " leaf hashes")
        a(cols * nb, what + ": one unit of its columns")
        f(cols * nb, what + ": one unit of its columns")
        a(4 * (nL - capl), what + " nodes")

    def chunks(what):
        a(chunk * n, what + ": monomials of a chunk")
        a(chunk * nb, what + ": one unit of a chunk")
        f(chunk * nb, what + ": one unit of a chunk")
        f(chunk * n, what + ": monomials of a chunk")

    tree_by_unit("setup tree", S)
    tree_by_unit("witness tree", W)
    a(n_s2 * n, "stage-2 columns (kept)")
    tree_by_unit("stage-2 tree", n_s2)
    a(2 * nQ, "gathered quotient")
    q_units = max(1, (Q << split) // world)
    if sharded:
        a(2 * q_units * nb, "this rank's quotient units")
    unit = (S + W + n_s2 + (2 if split else 0)) * nb
    a(unit, "one unit of every column the quotient reads")
    f(unit, "one unit of every column the quotient reads")
    if sharded:
        a(q_units * 2 * nb, "quotient exchange, send")
        a(world * q_units * 2 * nb, "quotient exchange, receive")
        f(world * q_units * 2 * nb, "quotient exchange, receive")
        f(q_units * 2 * nb, "quotient exchange, send")
        f(2 * q_units * nb, "this rank's quotient units")
    a(2 * nQ, "quotient chunks")
    f(2 * nQ, "gathered quotient")
    a(2 * Q * nL, "quotient LDE")
    f(2 * nQ, "quotient chunks")
    tree("quotient tree")
    chunks("openings from local slot 0")
    a(2 * nL, "DEEP codeword")
    chunks("DEEP on this rank's units of cosets [0, L)")
    sched, nq = _schedule(bj, log_n, L, cap)
    log_m = log_n + L.bit_length() - 1
    for k in sched:
        lv = (1 << (log_m - k)) // world
        a(4 * lv, "FRI leaf hashes")
        a(4 * (lv - capl), "FRI nodes")
        a(lv, "FRI folded c0")
        a(lv, "FRI folded c1")
        log_m -= k
    fft = 1 << log_m
    a(fft, "FRI last codeword c0")
    a(fft, "FRI last codeword c1")
    if sharded:
        a(2 * fft // world, "FRI last codeword, send")
        a(2 * fft, "FRI last codeword, receive")
        f(2 * fft, "FRI last codeword, receive")
        f(2 * fft // world, "FRI last codeword, send")
    f(fft, "FRI last codeword c0")
    f(fft, "FRI last codeword c1")
    depth = 0
    while (nL >> depth) > capl:
        depth += 1
    row = max(2 * Q, 4 * depth, 2 << max(sched))  # no row of the setup, witness and stage-2 oracles is gathered from a kept unit
    a(nq * row, "query gather")
    f(nq * row, "query gather")
    a(chunk * n, "query rows: monomials of a chunk")
    a(chunk * nb, "query rows: one unit of a chunk")
    a(nq * chunk, "query rows: gather of a chunk")
    return ev


def _peak(ev):
    cur = peak = 0
    for sign, cnt, _ in ev:
        cur += (1 if sign == "+" else -1) * 8 * max(cnt, 1)
        assert cur >= 0
        peak = max(peak, cur)
    return peak


def _reserve(log_n, Q, L):
    """what the library keeps outside the pool: twiddles, coset-power tables, NTT scratch, parameter arena (every plan)"""
    n, D = 1 << log_n, max(L, Q)
    log_d = D.bit_length() - 1
    return (8 * n * D + min(3 << 30, 8 * n * (D + Q + 2)) + 64 * 16 * (1 << ((log_n + log_d + 2) // 2)) + 8 * max(1 << 27, 4 * n)
            + (16 << 20))


def _circuit(bj, log_n, V, C, Q, L, cap, lookup):
    c = bj.native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree, c.fri_lde_factor, c.merkle_tree_cap_size = log_n, V, C, Q, L, cap
    c.security_level = 100
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup
    return c


def _owns_no_quotient_unit(world, Q, L):
    """Q < L and more ranks than quotient units: the plan does not apply (0)"""
    split = max(0, world.bit_length() - L.bit_length())
    return (Q << split) < world


def _native(bj, fn, world, log_n, V, C, Q, L, cap, lookup):
    out = ctypes.c_uint64(1)
    c = _circuit(bj, log_n, V, C, Q, L, cap, lookup)
    status = getattr(bj.native.lib, fn)(ctypes.byref(c), world, ctypes.byref(out))
    return status, out.value


def _sharded(bj, world, log_n, V, C, Q, L, cap, lookup):
    status, v = _native(bj, "bj_proof_memory_plan_recompute_sharded", world, log_n, V, C, Q, L, cap, lookup)
    assert status == 0
    return v


def _plan(bj, world, log_n, V, C, Q, L, cap, lookup):
    lk = dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None
    return bj.proof_memory_plan(log_n, V, C, Q, _cfg(L, cap), lookup=lk, world=world)


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("log_n", [12, 20, 22, 23])
def test_world_one_is_the_single_gpu_recompute_plan(bj, shape, log_n):
    V, C, Q, L, cap, lookup = SHAPES[shape]
    status, one = _native(bj, "bj_proof_memory_plan_recompute", 1, log_n, *SHAPES[shape])
    assert status == 0 and one > 0
    assert _sharded(bj, 1, log_n, *SHAPES[shape]) == one
    lk = dict(width=lookup[0], num_repetitions=lookup[1])
    assert bj.proof_memory_plan_recompute_sharded(log_n, V, C, Q, _cfg(L, cap), 1, lookup=lk) == one


@pytest.mark.parametrize("log_n,V,C,Q,L,cap,lookup", [
    (9, 20, 6, 8, 2, 16, None), (10, 155, 8, 8, 2, 32, (3, 8)), (11, 20, 6, 4, 2, 8, (4, 2)), (12, 40, 6, 4, 8, 16, None),
    (10, 20, 6, 4, 4, 8, (4, 2)), (12, 60, 7, 8, 4, 32, None), (10, 20, 6, 2, 4, 8, (4, 2)), (13, 92, 7, 4, 8, 16, (4, 8))])
@pytest.mark.parametrize("world", [1, 2, 4, 8, 16])
def test_recompute_sharded_plan_is_the_sum_of_the_driver_allocations(bj, world, log_n, V, C, Q, L, cap, lookup):
    if cap < world or world > 8 * L:
        pytest.skip("no sharded context of this world for this cap / LDE factor")
    got = _sharded(bj, world, log_n, V, C, Q, L, cap, lookup)
    if _owns_no_quotient_unit(world, Q, L):
        assert got == 0
        return
    assert got == _peak(_recompute_sharded_allocations(bj, log_n, V, C, Q, L, cap, lookup, world)) + _reserve(log_n, Q, L)


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("log_n", [20, 22, 23, 24])
@pytest.mark.parametrize("world", [2, 4, 8, 16])
def test_below_the_sharded_streamed_and_resident_plans(bj, shape, log_n, world):
    V, C, Q, L, cap, lookup = SHAPES[shape]
    if cap < world or world > 8 * L:
        pytest.skip("no sharded context of this world for this cap / LDE factor")
    got = _sharded(bj, world, log_n, *SHAPES[shape])
    if _owns_no_quotient_unit(world, Q, L):
        assert got == 0
        return
    plan = _plan(bj, world, log_n, *SHAPES[shape])
    assert plan["recompute"] is None                 # bj_proof_memory_plan_recompute keeps its one-GPU meaning
    assert 0 < got < plan["resident"], (got, plan)
    if plan["streamed_sharded"]:
        assert got < plan["streamed_sharded"], (got, plan)


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("log_n", [22, 23, 24])
def test_shrinks_as_the_world_grows(bj, shape, log_n):
    """the per-rank plan falls with the world until what every rank holds whole - the natural-order stage-2 columns and the
    gathered quotient, 8 n (n_s2 + 4 Q) bytes - dominates it; it never grows"""
    V, C, Q, L, cap, lookup = SHAPES[shape]
    worlds = [w for w in (1, 2, 4, 8, 16) if w <= cap and w <= 8 * L and not _owns_no_quotient_unit(w, Q, L)]
    per_rank = [_sharded(bj, w, log_n, *SHAPES[shape]) for w in worlds]
    assert all(b <= a for a, b in zip(per_rank, per_rank[1:])), per_rank
    assert per_rank[1] < per_rank[0], per_rank
    n = 1 << log_n
    n_s2 = 2 + 2 * ((V + Q - 1) // Q - 1) + 2 * (lookup[1] + 1)
    whole = 8 * n * (n_s2 + 4 * Q) + _reserve(log_n, Q, L)
    assert per_rank[-1] > whole


def test_production_shape_2p23_on_two_gpus_is_below_one_gpu(bj):
    """at 2^23 rows two ranks on the streamed plan need more per device than one GPU on the recompute plan; two ranks on the
    recompute plan need less"""
    p = SHAPES["production"]
    one = _sharded(bj, 1, 23, *p)
    two = _sharded(bj, 2, 23, *p)
    assert _plan(bj, 2, 23, *p)["streamed_sharded"] > one
    assert two < one < 80 * GB


def test_rejects_the_shapes_sharding_rejects(bj):
    fn = "bj_proof_memory_plan_recompute_sharded"
    assert _native(bj, fn, 32, 12, 20, 6, 8, 2, 16, None) == (INVALID_ARG, 0)    # cap below world
    assert _native(bj, fn, 32, 12, 20, 6, 8, 2, 64, None) == (INVALID_ARG, 0)    # world > 8 * LDE factor
    assert _native(bj, fn, 16, 3, 20, 6, 8, 2, 32, None) == (INVALID_ARG, 0)     # 8 row blocks of 1 row
    assert _native(bj, fn, 3, 12, 20, 6, 8, 2, 16, None) == (INVALID_ARG, 0)     # world not a power of two
    assert _native(bj, fn, 16, 12, 20, 6, 8, 2, 32, None)[0] == 0
    assert _native(bj, fn, 8, 12, 20, 6, 4, 8, 16, None) == (0, 0)              # Q < L: ranks 4-7 own no quotient unit
    assert _native(bj, fn, 4, 12, 20, 6, 4, 8, 16, None)[1] > 0
    c = _circuit(bj, 12, 20, 6, 8, 2, 16, None)
    assert bj.native.lib.bj_proof_memory_plan_recompute_sharded(ctypes.byref(c), 2, None) == INVALID_ARG
    from era_boojum_b200 import BoojumError
    with pytest.raises(BoojumError):
        bj.proof_memory_plan_recompute_sharded(12, 20, 6, 8, _cfg(2, 16), 32)
