"""bj_proof_memory_plan_streamed_sharded (no GPU): the streamed plan on each rank of a sharded context, counted from the
circuit's shapes.  With quotient degree Q above the LDE factor L, every rank evaluates the setup, witness and stage-2 columns
on its units of the committed cosets [0, L) only, and its quotient units of cosets [L, Q) one at a time into a unit-sized
scratch (whole cosets on a coset shard, world <= L; row blocks of n / B rows on a split shard, world = L * B, with their
z(omega x) columns).  The plan is checked against the driver's pool allocations on one rank, listed here one by one in the
order prover.cu makes them, against the sharded resident plan, and against the single-GPU streamed plan at world 1."""
import ctypes

import pytest

GB = 10**9

PRODUCTION = dict(log_n=22, V=155, C=8, Q=8, L=2, cap=32, lookup=(3, 8))


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


def _lde_columns(a, f, cols, n, world):
    """lde_columns on a sharded context: column groups of monomials, each all-gathered; group g + 1 is allocated before
    group g is released"""
    if world == 1 or cols < 2:
        return
    group = max(world, -(-(-(-cols // 4)) // world) * world)
    sizes = []
    for c0 in range(0, cols, group):
        cnt = min(group, cols - c0)
        sizes.append(world * -(-cnt // world) * n)
    for i, s in enumerate(sizes):
        a(s, "monomials of column group %d" % i)
        if i:
            f(sizes[i - 1], "monomials of column group %d" % (i - 1))
    f(sizes[-1], "monomials of column group %d" % (len(sizes) - 1))


def _streamed_sharded_allocations(bj, log_n, V, C, Q, L, cap, lookup, world):
    """the streamed driver's pool allocations on one rank of `world`, in order: ("+" | "-", u64 count, what)"""
    n = 1 << log_n
    split = max(0, world.bit_length() - L.bit_length())   # log2(B), B = world / L row blocks per coset when world > L
    nb = n >> split
    T = lookup[0] + 1 if lookup else 0
    S, W = V + C + T, V + (1 if lookup else 0)
    n_s2 = 2 + 2 * ((V + Q - 1) // Q - 1) + (2 * (lookup[1] + 1) if lookup else 0)
    nL, nQ = n * L // world, n * Q               # nL: this rank's part of a committed column
    capl = cap // world
    ev = []
    a = lambda cnt, what: ev.append(("+", cnt, what))
    f = lambda cnt, what: ev.append(("-", cnt, what))

    def tree(what, leaves=nL):
        a(4 * leaves, what + " leaf hashes")
        a(4 * (leaves - capl), what + " nodes")

    a(S * nL, "setup LDE, this rank's units of cosets [0, L)")
    for cols in (V, C, T):
        _lde_columns(a, f, cols, n, world)
    tree("setup tree")
    a(V * nL, "witness LDE")
    _lde_columns(a, f, V, n, world)
    if lookup:
        a(nL, "multiplicities LDE")
    tree("witness tree")
    a(n_s2 * n, "stage-2 columns (kept)")
    a(n_s2 * nL, "stage-2 LDE")
    _lde_columns(a, f, n_s2, n, world)
    tree("stage-2 tree")
    a(2 * nQ, "gathered quotient")
    q_units = (Q << split) // world
    sharded = world > 1                          # one GPU writes the quotient straight into the gathered buffer
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
    a(2 * nL, "DEEP codeword")
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
    row = max(S, W, n_s2, 2 * Q, 4 * depth, 2 << max(sched))
    a(nq * row, "query gather")
    f(nq * row, "query gather")
    return ev


def _peak(ev):
    cur = peak = 0
    for sign, cnt, _ in ev:
        cur += (1 if sign == "+" else -1) * 8 * max(cnt, 1)
        assert cur >= 0
        peak = max(peak, cur)
    return peak


def _reserve(log_n, Q, L):
    """what the library keeps outside the pool: twiddles, coset-power tables, NTT scratch, parameter arena"""
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


def _sharded(bj, world, log_n, V, C, Q, L, cap, lookup):
    out = ctypes.c_uint64(1)
    c = _circuit(bj, log_n, V, C, Q, L, cap, lookup)
    assert bj.native.lib.bj_proof_memory_plan_streamed_sharded(ctypes.byref(c), world, ctypes.byref(out)) == 0
    return out.value


def _plan(bj, world, log_n, V, C, Q, L, cap, lookup):
    lk = dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None
    return bj.proof_memory_plan(log_n, V, C, Q, _cfg(L, cap), lookup=lk, world=world)


@pytest.mark.parametrize("world", [2, 4, 8, 16])
def test_production_shape_has_a_sharded_streamed_plan(bj, world):
    p = PRODUCTION
    got = _sharded(bj, world, **p)
    assert got > 0
    plan = _plan(bj, world, **p)
    assert plan["streamed_sharded"] == got
    assert plan["streamed"] is None                 # bj_proof_memory_plan_streamed keeps its one-GPU meaning
    assert got < plan["resident"]


@pytest.mark.parametrize("log_n", [22, 23])
def test_sharded_streamed_plan_does_not_grow_with_world(bj, log_n):
    p = dict(PRODUCTION, log_n=log_n)
    per_rank = [_sharded(bj, w, **p) for w in (1, 2, 4, 8, 16)]
    assert all(b <= a for a, b in zip(per_rank, per_rank[1:])), per_rank
    for w, b in zip((2, 4, 8, 16), per_rank[1:]):
        assert b < _plan(bj, w, **p)["resident"], w


def test_production_shape_2p23_fits_two_80gb_devices_only_on_the_streamed_plan(bj):
    p = dict(PRODUCTION, log_n=23)
    plan = _plan(bj, 2, **p)
    assert plan["resident"] > 80 * GB
    assert plan["streamed_sharded"] < 80 * GB


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("Q,L", [(2, 2), (4, 4), (8, 8), (2, 4), (4, 8)])
def test_no_sharded_streamed_plan_when_the_quotient_degree_is_at_most_the_lde_factor(bj, world, Q, L):
    assert _sharded(bj, world, 10, 20, 6, Q, L, 16, (4, 2)) == 0
    assert _plan(bj, world, 10, 20, 6, Q, L, 16, (4, 2))["streamed_sharded"] is None


@pytest.mark.parametrize("log_n,V,C,Q,L,cap,lookup", [
    (9, 20, 6, 8, 2, 16, None), (10, 155, 8, 8, 2, 32, (3, 8)), (11, 20, 6, 4, 2, 8, (4, 2)), (12, 40, 6, 4, 2, 16, None),
    (10, 20, 6, 8, 4, 16, (4, 2)), (12, 60, 7, 8, 4, 32, None), (13, 155, 8, 8, 2, 32, (3, 8))])
@pytest.mark.parametrize("world", [1, 2, 4, 8, 16])
def test_sharded_streamed_plan_is_the_sum_of_the_driver_allocations(bj, world, log_n, V, C, Q, L, cap, lookup):
    if cap < world or world > 8 * L:
        pytest.skip("no sharded context of this world for this cap / LDE factor")
    got = _sharded(bj, world, log_n, V, C, Q, L, cap, lookup)
    assert got == _peak(_streamed_sharded_allocations(bj, log_n, V, C, Q, L, cap, lookup, world)) + _reserve(log_n, Q, L)
    # a rank with two quotient units (Q = 2 L) keeps one and evaluates the other into a scratch of the same size: no saving
    split = max(0, world.bit_length() - L.bit_length())
    if (Q << split) // world >= 4:
        assert got < _plan(bj, world, log_n, V, C, Q, L, cap, lookup)["resident"]


@pytest.mark.parametrize("log_n,V,C,Q,L,cap,lookup", [
    (9, 20, 6, 8, 2, 16, None), (10, 155, 8, 8, 2, 32, (3, 8)), (11, 20, 6, 4, 2, 8, (4, 2)), (10, 20, 6, 8, 4, 16, (4, 2)),
    (22, 155, 8, 8, 2, 32, (3, 8))])
def test_world_one_is_the_single_gpu_streamed_plan(bj, log_n, V, C, Q, L, cap, lookup):
    out = ctypes.c_uint64()
    c = _circuit(bj, log_n, V, C, Q, L, cap, lookup)
    assert bj.native.lib.bj_proof_memory_plan_streamed(ctypes.byref(c), 1, ctypes.byref(out)) == 0
    assert out.value > 0 and _sharded(bj, 1, log_n, V, C, Q, L, cap, lookup) == out.value


def test_sharded_streamed_plan_rejects_bad_shapes(bj):
    lib = bj.native.lib
    c = _circuit(bj, 10, 20, 6, 3, 2, 16, None)
    out = ctypes.c_uint64()
    assert lib.bj_proof_memory_plan_streamed_sharded(ctypes.byref(c), 2, ctypes.byref(out)) == -1   # Q not a power of two
    c.quotient_degree = 8
    assert lib.bj_proof_memory_plan_streamed_sharded(ctypes.byref(c), 3, ctypes.byref(out)) == -1  # world not a power of two
    assert lib.bj_proof_memory_plan_streamed_sharded(ctypes.byref(c), 32, ctypes.byref(out)) == -1  # cap below world
    assert lib.bj_proof_memory_plan_streamed_sharded(ctypes.byref(c), 2, None) == -1
