"""bj_proof_memory_plan (no GPU): the device bytes of bj_setup_create + bj_prove at their peak, counted from the circuit's shapes.
The 2^22-row bench shape does not fit an 80 GB device on the resident plan and fits well on the compact one; at small shapes
the plan is checked against the driver's pool allocations, listed here one by one in the order prover.cu makes them."""
import ctypes

import pytest

GB = 10**9


@pytest.fixture(scope="module")
def bj():
    import era_boojum_b200 as m
    return m


def _cfg(bj, L, cap=16):
    from era_boojum_b200 import prover
    return prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100)


def _schedule(bj, log_n, L, cap):
    lib = bj.native.lib
    new_pow, nq, sl, fd = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    sched = (ctypes.c_uint32 * 32)()
    assert lib.bj_compute_fri_schedule(100, cap, 0, L.bit_length() - 1, log_n, ctypes.byref(new_pow), ctypes.byref(nq), sched,
                                       ctypes.byref(sl), ctypes.byref(fd)) == 0
    return list(sched[:sl.value]), nq.value


def _allocations(bj, log_n, V, C, Q, L, cap, lookup, compact, chunk=2):
    """the driver's pool allocations in order: ("+" | "-", u64 count, what).  lookup: (width, repetitions) or None."""
    n = 1 << log_n
    D = max(L, Q)
    T = lookup[0] + 1 if lookup else 0
    S, W = V + C + T, V + (1 if lookup else 0)
    n_s2 = 2 + 2 * ((V + Q - 1) // Q - 1) + (2 * (lookup[1] + 1) if lookup else 0)
    leaves, nD, nL, nQ, Qn = n * L, n * D, n * L, n * Q, n * Q
    ev = []
    a = lambda cnt, what: ev.append(("+", cnt, what))
    f = lambda cnt, what: ev.append(("-", cnt, what))

    def tree(what):
        a(4 * leaves, what + " leaf hashes")
        a(4 * (leaves - cap), what + " nodes")

    a(S * nD, "setup LDE")
    tree("setup tree")
    if compact:
        a(S * Qn, "setup cosets [0, Q)")
        f(S * nD, "setup LDE")
    # the compact plan holds the witness and stage-2 LDEs as up to 4 column groups and repacks them group by group
    groups = lambda cols: [min(-(-cols // 4), cols - c0) for c0 in range(0, cols, -(-cols // 4))]
    wg = (groups(V) + ([1] if lookup else [])) if compact else [V] + ([1] if lookup else [])
    for g in wg:
        a(g * nD, "witness LDE group")
    tree("witness tree")
    if compact:
        for g in wg:
            a(g * Qn, "witness group cosets [0, Q)")
            f(g * nD, "witness LDE group")
    sg = groups(n_s2) if compact else [n_s2]
    a(n_s2 * n, "stage-2 columns")
    for g in sg:
        a(g * nD, "stage-2 LDE group")
    if not compact:
        f(n_s2 * n, "stage-2 columns")
    tree("stage-2 tree")
    if compact:
        for g in sg:
            a(g * Qn, "stage-2 group cosets [0, Q)")
            f(g * nD, "stage-2 LDE group")
    a(2 * nQ, "quotient cosets")
    a(2 * nQ, "quotient chunks")
    f(2 * nQ, "quotient cosets")
    a(2 * Q * nL, "quotient LDE")
    f(2 * nQ, "quotient chunks")
    tree("quotient tree")
    a(2 * nL, "DEEP codeword")
    if compact:
        a(chunk * n, "recompute monomials")
        a(chunk * n, "recompute coset")
        f(chunk * n, "recompute monomials")
        f(chunk * n, "recompute coset")
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
    while (leaves >> depth) > cap:
        depth += 1
    row = max(S, W, n_s2, 2 * Q, 4 * depth, 2 << max(sched))
    a(nq * row, "query gather")
    f(nq * row, "query gather")
    if compact:
        a(chunk * n, "recompute monomials")
        a(chunk * n, "recompute coset")
        a(nq * chunk, "recomputed rows")
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


def test_bench_shape_2p22_needs_the_compact_plan_on_80gb(bj):
    """the 2^22-row SHA-shaped bench circuit: 92 copy-permutation columns, 7 constants, 8 lookups of width 4, Q = 4, L = 8"""
    plan = bj.proof_memory_plan(22, 92, 7, 4, _cfg(bj, 8), lookup=dict(width=4, num_repetitions=8))
    assert plan["resident"] > 80 * GB
    assert plan["compact"] < 0.8 * 80 * GB
    # the default 2^21 bench proof keeps the resident plan on an 80 GB device
    assert bj.proof_memory_plan(21, 92, 7, 4, _cfg(bj, 8), lookup=dict(width=4, num_repetitions=8))["resident"] < 60 * GB


@pytest.mark.parametrize("log_n,V,C,Q,L,cap,lookup", [
    (9, 20, 6, 4, 8, 16, None), (10, 60, 7, 4, 8, 16, (4, 8)), (12, 20, 6, 2, 4, 8, (4, 2)), (11, 40, 6, 4, 8, 16, (4, 2)),
    (10, 20, 6, 8, 2, 32, None)])
def test_plan_is_the_sum_of_the_driver_allocations(bj, log_n, V, C, Q, L, cap, lookup):
    lk = dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None
    plan = bj.proof_memory_plan(log_n, V, C, Q, _cfg(bj, L, cap), lookup=lk)
    reserve = _reserve(log_n, Q, L)
    assert plan["resident"] == _peak(_allocations(bj, log_n, V, C, Q, L, cap, lookup, False)) + reserve
    if Q >= L:
        assert plan["compact"] is None
        return
    compact = _peak(_allocations(bj, log_n, V, C, Q, L, cap, lookup, True)) + reserve
    assert plan["compact"] == compact
    assert plan["compact"] < plan["resident"]


def test_no_compact_plan_on_several_gpus(bj):
    plan = bj.proof_memory_plan(14, 60, 6, 4, _cfg(bj, 8), world=2)
    assert plan["compact"] is None and plan["resident"] > 0
    # each of the world GPUs holds 1 / world of the LDE: the per-GPU plan shrinks
    assert plan["resident"] < bj.proof_memory_plan(14, 60, 6, 4, _cfg(bj, 8))["resident"]


def test_plan_rejects_bad_shapes(bj):
    with pytest.raises(bj.BoojumError):
        bj.proof_memory_plan(10, 20, 6, 3, _cfg(bj, 8))            # quotient degree not a power of two
    with pytest.raises(bj.BoojumError):
        bj.proof_memory_plan(10, 20, 6, 4, _cfg(bj, 8), world=3)
