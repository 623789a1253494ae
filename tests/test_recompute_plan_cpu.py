"""bj_proof_memory_plan_recompute (no GPU): the recompute plan's device bytes, counted from the circuit's shapes.  The plan keeps
no coset of the setup, witness and stage-2 columns: the trees are built one coset at a time, and the quotient, openings, DEEP
and query answers rebuild the cosets they read.  It applies on one GPU to any quotient degree, and is checked against the
driver's pool allocations, listed here one by one in the order prover.cu makes them, and against the other plans."""
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


def _recompute_allocations(bj, log_n, V, C, Q, L, cap, lookup, chunk=2):
    """the recompute driver's pool allocations in order: ("+" | "-", u64 count, what).  lookup: (width, repetitions) or None."""
    n = 1 << log_n
    T = lookup[0] + 1 if lookup else 0
    S, W = V + C + T, V + (1 if lookup else 0)
    n_s2 = 2 + 2 * ((V + Q - 1) // Q - 1) + (2 * (lookup[1] + 1) if lookup else 0)
    nL, nQ = n * L, n * Q
    ev = []
    a = lambda cnt, what: ev.append(("+", cnt, what))
    f = lambda cnt, what: ev.append(("-", cnt, what))

    def tree(what):
        a(4 * nL, what + " leaf hashes")
        a(4 * (nL - cap), what + " nodes")

    def tree_by_coset(what, cols):
        a(4 * nL, what + " leaf hashes")
        a(cols * n, what + ": one coset of its columns")
        f(cols * n, what + ": one coset of its columns")
        a(4 * (nL - cap), what + " nodes")

    def chunks(what):
        a(chunk * n, what + ": monomials of a chunk")
        a(chunk * n, what + ": one coset of a chunk")
        f(chunk * n, what + ": monomials of a chunk")
        f(chunk * n, what + ": one coset of a chunk")

    tree_by_coset("setup tree", S)
    tree_by_coset("witness tree", W)
    a(n_s2 * n, "stage-2 columns (kept)")
    tree_by_coset("stage-2 tree", n_s2)
    a(2 * nQ, "quotient cosets")
    a((S + W + n_s2) * n, "one coset of every column the quotient reads")
    f((S + W + n_s2) * n, "one coset of every column the quotient reads")
    a(2 * nQ, "quotient chunks")
    f(2 * nQ, "quotient cosets")
    a(2 * Q * nL, "quotient LDE")
    f(2 * nQ, "quotient chunks")
    tree("quotient tree")
    chunks("openings from coset 0")
    a(2 * nL, "DEEP codeword")
    chunks("DEEP on cosets [0, L)")
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
    row = max(2 * Q, 4 * depth, 2 << max(sched))  # no row of the setup, witness and stage-2 oracles is gathered from a kept coset
    a(nq * row, "query gather")
    f(nq * row, "query gather")
    a(chunk * n, "query rows: monomials of a chunk")
    a(chunk * n, "query rows: one coset of a chunk")
    a(nq * chunk, "query rows: gather of a chunk")
    return ev


def _peak(ev):
    cur = peak = 0
    for sign, cnt, _ in ev:
        cur += (1 if sign == "+" else -1) * 8 * max(cnt, 1)
        peak = max(peak, cur)
    return peak


def _reserve(log_n, Q, L):
    """what the library keeps outside the pool: twiddles, coset-power tables, NTT scratch, parameter arena (every plan)"""
    n, D = 1 << log_n, max(L, Q)
    log_d = D.bit_length() - 1
    return (8 * n * D + min(3 << 30, 8 * n * (D + Q + 2)) + 64 * 16 * (1 << ((log_n + log_d + 2) // 2)) + 8 * max(1 << 27, 4 * n)
            + (16 << 20))


def _plan(bj, log_n, V, C, Q, L, cap, lookup, world=1):
    lk = dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None
    return bj.proof_memory_plan(log_n, V, C, Q, _cfg(L, cap), lookup=lk, world=world)


def _circuit(bj, log_n, V, C, Q, L, cap, lookup):
    c = bj.native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree, c.fri_lde_factor, c.merkle_tree_cap_size = log_n, V, C, Q, L, cap
    c.security_level = 100
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup
    return c


# the production shape (155 columns, 8 constants, 8 lookups of width 3, Q = 8 over L = 2, cap 32), the bench shape (60 columns
# and the 32 its 8 lookups of width 4 read, 7 constants, Q = 4 over L = 8, cap 16) and a Q = L shape
SHAPES = {"production": (155, 8, 8, 2, 32, (3, 8)), "bench": (92, 7, 4, 8, 16, (4, 8)), "q_equals_l": (92, 7, 4, 4, 16, (4, 8))}


@pytest.mark.parametrize("log_n,V,C,Q,L,cap,lookup", [
    (9, 20, 6, 8, 2, 16, None), (10, 155, 8, 8, 2, 32, (3, 8)), (11, 20, 6, 4, 2, 8, (4, 2)), (12, 40, 6, 4, 8, 16, None),
    (10, 20, 6, 4, 4, 8, (4, 2)), (12, 60, 7, 8, 4, 16, None), (10, 20, 6, 2, 4, 8, (4, 2))])
def test_recompute_plan_is_the_sum_of_the_driver_allocations(bj, log_n, V, C, Q, L, cap, lookup):
    plan = _plan(bj, log_n, V, C, Q, L, cap, lookup)
    assert plan["recompute"] == _peak(_recompute_allocations(bj, log_n, V, C, Q, L, cap, lookup)) + _reserve(log_n, Q, L)


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("log_n", [20, 21, 22, 23])
def test_recompute_plan_is_below_every_other_plan(bj, shape, log_n):
    plan = _plan(bj, log_n, *SHAPES[shape])
    others = [plan[k] for k in ("resident", "compact", "streamed") if plan[k]]
    assert others and plan["recompute"] < min(others), plan


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_recompute_plan_grows_with_log_n(bj, shape):
    sizes = [_plan(bj, log_n, *SHAPES[shape])["recompute"] for log_n in range(16, 25)]
    assert all(a < b for a, b in zip(sizes, sizes[1:])), sizes


def test_production_shape_2p23_fits_one_80gb_device_with_its_inputs(bj):
    """at 2^23 rows the production shape's natural-order inputs (155 variables and sigmas, 8 constants, 4 tables, the
    multiplicities) and the recompute plan fit one 80 GB device together; the streamed plan alone does not"""
    plan = _plan(bj, 23, *SHAPES["production"])
    inputs = 8 * (1 << 23) * (155 + 155 + 8 + 4 + 1)
    assert plan["streamed"] > 80 * GB
    assert plan["recompute"] + inputs < 0.8 * 80 * GB


@pytest.mark.parametrize("world", [2, 4, 8])
def test_no_recompute_plan_on_several_gpus(bj, world):
    assert _plan(bj, 12, 20, 6, 8, 2, 32, None, world=world)["recompute"] is None
    out = ctypes.c_uint64(1)
    c = _circuit(bj, 12, 20, 6, 8, 2, 32, None)
    assert bj.native.lib.bj_proof_memory_plan_recompute(ctypes.byref(c), world, ctypes.byref(out)) == 0 and out.value == 0
    assert bj.native.lib.bj_proof_memory_plan_recompute(ctypes.byref(c), 1, ctypes.byref(out)) == 0 and out.value > 0


def test_recompute_plan_rejects_bad_shapes(bj):
    c = _circuit(bj, 10, 20, 6, 3, 2, 16, None)
    out = ctypes.c_uint64()
    assert bj.native.lib.bj_proof_memory_plan_recompute(ctypes.byref(c), 1, ctypes.byref(out)) == -1   # Q not a power of two
    c.quotient_degree = 8
    assert bj.native.lib.bj_proof_memory_plan_recompute(ctypes.byref(c), 3, ctypes.byref(out)) == -1
    assert bj.native.lib.bj_proof_memory_plan_recompute(ctypes.byref(c), 1, None) == -1
