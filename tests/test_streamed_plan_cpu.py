"""bj_proof_memory_plan_streamed (no GPU): the streamed plan's device bytes, counted from the circuit's shapes.  With quotient
degree Q above the LDE factor L, the setup, witness and stage-2 columns are evaluated on cosets [0, L) only and the quotient
evaluates every column it reads onto one coset of [L, Q) at a time.  The plan is checked against the driver's pool allocations,
listed here one by one in the order prover.cu makes them, and against the resident plan."""
import ctypes

import pytest

GB = 10**9


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


def _streamed_allocations(bj, log_n, V, C, Q, L, cap, lookup):
    """the streamed driver's pool allocations in order: ("+" | "-", u64 count, what).  lookup: (width, repetitions) or None."""
    n = 1 << log_n
    T = lookup[0] + 1 if lookup else 0
    S, W = V + C + T, V + (1 if lookup else 0)
    n_s2 = 2 + 2 * ((V + Q - 1) // Q - 1) + (2 * (lookup[1] + 1) if lookup else 0)
    nL, nQ = n * L, n * Q
    ev = []
    a = lambda cnt, what: ev.append(("+", cnt, what))
    f = lambda cnt, what: ev.append(("-", cnt, what))

    def tree(what, leaves=nL):
        a(4 * leaves, what + " leaf hashes")
        a(4 * (leaves - cap), what + " nodes")

    a(S * nL, "setup LDE, cosets [0, L)")
    tree("setup tree")
    a(V * nL, "witness LDE, cosets [0, L)")
    if lookup:
        a(nL, "multiplicities LDE, cosets [0, L)")
    tree("witness tree")
    a(n_s2 * n, "stage-2 columns (kept)")
    a(n_s2 * nL, "stage-2 LDE, cosets [0, L)")
    tree("stage-2 tree")
    a(2 * nQ, "quotient cosets")
    a((S + W + n_s2) * n, "one coset of every column the quotient reads")
    f((S + W + n_s2) * n, "one coset of every column the quotient reads")
    a(2 * nQ, "quotient chunks")
    f(2 * nQ, "quotient cosets")
    a(2 * Q * nL, "quotient LDE")
    f(2 * nQ, "quotient chunks")
    tree("quotient tree")
    a(2 * nL, "DEEP codeword")
    sched, nq = _schedule(bj, log_n, L, cap)
    log_m = log_n + L.bit_length() - 1
    for k in sched:
        lv = 1 << (log_m - k)
        a(4 * lv, "FRI leaf hashes")
        a(4 * (lv - cap), "FRI nodes")
        a(lv, "FRI folded c0")
        a(lv, "FRI folded c1")
        log_m -= k
    a(1 << log_m, "FRI last codeword c0")
    a(1 << log_m, "FRI last codeword c1")
    f(1 << log_m, "FRI last codeword c0")
    f(1 << log_m, "FRI last codeword c1")
    depth = 0
    while (nL >> depth) > cap:
        depth += 1
    row = max(S, W, n_s2, 2 * Q, 4 * depth, 2 << max(sched))
    a(nq * row, "query gather")
    f(nq * row, "query gather")
    return ev


def _peak(ev):
    cur = peak = 0
    for sign, cnt, _ in ev:
        cur += (1 if sign == "+" else -1) * 8 * max(cnt, 1)
        peak = max(peak, cur)
    return peak


def _reserve(log_n, Q, L):
    """what the library keeps outside the pool: twiddles, coset-power tables, NTT scratch, parameter arena"""
    n, D = 1 << log_n, max(L, Q)
    log_d = D.bit_length() - 1
    return (8 * n * D + min(3 << 30, 8 * n * (D + Q + 2)) + 64 * 16 * (1 << ((log_n + log_d + 2) // 2)) + 8 * max(1 << 27, 4 * n)
            + (16 << 20))


def _plan(bj, log_n, V, C, Q, L, cap, lookup, world=1):
    lk = dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None
    return bj.proof_memory_plan(log_n, V, C, Q, _cfg(L, cap), lookup=lk, world=world)


@pytest.mark.parametrize("log_n,V,C,Q,L,cap,lookup", [
    (9, 20, 6, 8, 2, 16, None), (10, 155, 8, 8, 2, 32, (3, 8)), (11, 20, 6, 4, 2, 8, (4, 2)), (12, 40, 6, 4, 2, 8, None),
    (10, 20, 6, 8, 4, 16, (4, 2)), (12, 60, 7, 8, 4, 16, None)])
def test_streamed_plan_is_the_sum_of_the_driver_allocations(bj, log_n, V, C, Q, L, cap, lookup):
    plan = _plan(bj, log_n, V, C, Q, L, cap, lookup)
    assert plan["compact"] is None
    assert plan["streamed"] == _peak(_streamed_allocations(bj, log_n, V, C, Q, L, cap, lookup)) + _reserve(log_n, Q, L)
    assert plan["streamed"] < plan["resident"]


def test_production_shape_2p22_fits_one_80gb_device_on_the_streamed_plan(bj):
    """the production shape (155 copy-permutation columns, 8 constants, 8 lookups of width 3, Q = 8, L = 2, cap 32): the resident
    plan is above 80 GB at 2^22 rows, the streamed plan well below it"""
    plan = _plan(bj, 22, 155, 8, 8, 2, 32, (3, 8))
    assert plan["resident"] > 80 * GB
    assert plan["streamed"] < 0.7 * 80 * GB


@pytest.mark.parametrize("Q,L", [(2, 2), (4, 4), (8, 8), (2, 4), (4, 8)])
def test_no_streamed_plan_when_the_quotient_degree_is_at_most_the_lde_factor(bj, Q, L):
    assert _plan(bj, 10, 20, 6, Q, L, 16, (4, 2))["streamed"] is None


@pytest.mark.parametrize("world", [2, 4])
def test_no_streamed_plan_on_several_gpus(bj, world):
    plan = _plan(bj, 12, 20, 6, 8, 2, 32, None, world=world)
    assert plan["streamed"] is None and plan["resident"] > 0
    out = ctypes.c_uint64(1)
    c = bj.native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree, c.fri_lde_factor, c.merkle_tree_cap_size = 12, 20, 6, 8, 2, 32
    c.security_level = 100
    assert bj.native.lib.bj_proof_memory_plan_streamed(ctypes.byref(c), world, ctypes.byref(out)) == 0 and out.value == 0


def test_streamed_plan_rejects_bad_shapes(bj):
    c = bj.native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree, c.fri_lde_factor, c.merkle_tree_cap_size = 10, 20, 6, 3, 2, 16
    c.security_level = 100
    out = ctypes.c_uint64()
    assert bj.native.lib.bj_proof_memory_plan_streamed(ctypes.byref(c), 1, ctypes.byref(out)) == -1   # Q not a power of two
    c.quotient_degree = 8
    assert bj.native.lib.bj_proof_memory_plan_streamed(ctypes.byref(c), 3, ctypes.byref(out)) == -1
    assert bj.native.lib.bj_proof_memory_plan_streamed(ctypes.byref(c), 1, None) == -1
