"""bj_proof_memory_plan_recompute_blocks (no GPU): the one-GPU recompute plan with every coset cut into B row blocks in the trees
and the quotient.  Each tree is built one row block of n / B rows at a time, and the quotient evaluates every column it reads,
and z(omega x), onto one of the Q * B row blocks of cosets [0, Q) at a time, so both scratches fall by B.  At B = 1 the plan is
bj_proof_memory_plan_recompute.  Checked against the driver's pool allocations, listed here one by one in the order prover.cu
makes them, against the lane split of the plan, and against the shapes and block counts the plan refuses."""
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


def _lk(lookup):
    return dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None


def _blocks_plan(bj, log_n, V, C, Q, L, cap, lookup, blocks):
    return bj.proof_memory_plan_recompute_blocks(log_n, V, C, Q, _cfg(L, cap), blocks, lookup=_lk(lookup))


def _plan(bj, log_n, V, C, Q, L, cap, lookup):
    return bj.proof_memory_plan(log_n, V, C, Q, _cfg(L, cap), lookup=_lk(lookup))


def _circuit(bj, log_n, V, C, Q, L, cap, lookup):
    c = bj.native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree, c.fri_lde_factor, c.merkle_tree_cap_size = log_n, V, C, Q, L, cap
    c.security_level = 100
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup
    return c


def _schedule(bj, log_n, L, cap):
    lib = bj.native.lib
    new_pow, nq, sl, fd = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    sched = (ctypes.c_uint32 * 32)()
    assert lib.bj_compute_fri_schedule(100, cap, 0, L.bit_length() - 1, log_n, ctypes.byref(new_pow), ctypes.byref(nq), sched,
                                       ctypes.byref(sl), ctypes.byref(fd)) == 0
    return list(sched[:sl.value]), nq.value


def _allocations(bj, log_n, V, C, Q, L, cap, lookup, B, chunk=2):
    """the recompute driver's pool allocations with B row blocks per coset, in order: ("+" | "-", u64 count, what)"""
    n = 1 << log_n
    nb = n // B
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

    def tree_by_block(what, cols):
        a(4 * nL, what + " leaf hashes")
        a(cols * nb, what + ": one row block of its columns")
        f(cols * nb, what + ": one row block of its columns")
        a(4 * (nL - cap), what + " nodes")

    def chunks(what):  # the openings and DEEP rebuild whole cosets whatever B is
        a(chunk * n, what + ": monomials of a chunk")
        a(chunk * n, what + ": one coset of a chunk")
        f(chunk * n, what + ": monomials of a chunk")
        f(chunk * n, what + ": one coset of a chunk")

    tree_by_block("setup tree", S)
    tree_by_block("witness tree", W)
    a(n_s2 * n, "stage-2 columns (kept)")
    tree_by_block("stage-2 tree", n_s2)
    a(2 * nQ, "quotient cosets")
    zn = 2 if B > 1 else 0  # a row block does not hold z(omega x): two more columns per unit
    a((S + W + n_s2 + zn) * nb, "one row block of every column the quotient reads")
    f((S + W + n_s2 + zn) * nb, "one row block of every column the quotient reads")
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
    a(nq * max(2 * Q, 4 * depth, 2 << max(sched)), "query gather")
    f(nq * max(2 * Q, 4 * depth, 2 << max(sched)), "query gather")
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


# the production shape (155 columns, 8 constants, 8 lookups of width 3, Q = 8 over L = 2, cap 32), the bench shape (60 columns
# and the 32 its 8 lookups of width 4 read, 7 constants, Q = 4 over L = 8, cap 16) and a Q = L shape
SHAPES = {"production": (155, 8, 8, 2, 32, (3, 8)), "bench": (92, 7, 4, 8, 16, (4, 8)), "q_equals_l": (92, 7, 4, 4, 16, (4, 8))}


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("log_n", [10, 16, 20, 23, 24])
def test_one_block_is_the_recompute_plan(bj, shape, log_n):
    assert _blocks_plan(bj, log_n, *SHAPES[shape], 1) == _plan(bj, log_n, *SHAPES[shape])["recompute"]


@pytest.mark.parametrize("log_n,V,C,Q,L,cap,lookup", [
    (9, 20, 6, 8, 2, 16, None), (10, 155, 8, 8, 2, 32, (3, 8)), (11, 20, 6, 4, 2, 8, (4, 2)), (12, 40, 6, 4, 8, 16, None),
    (10, 20, 6, 4, 4, 8, (4, 2)), (12, 60, 7, 8, 4, 16, None), (10, 20, 6, 2, 4, 8, (4, 2)), (20, 155, 8, 8, 2, 32, (3, 8))])
@pytest.mark.parametrize("B", [1, 2, 4, 8])
def test_plan_is_the_peak_of_the_driver_allocations(bj, log_n, V, C, Q, L, cap, lookup, B):
    """the pool part of the plan (the library's reserve outside the pool does not depend on B) is the replayed peak"""
    reserve = _plan(bj, log_n, V, C, Q, L, cap, lookup)["recompute"] - _peak(_allocations(bj, log_n, V, C, Q, L, cap, lookup, 1))
    assert _blocks_plan(bj, log_n, V, C, Q, L, cap, lookup, B) == _peak(_allocations(bj, log_n, V, C, Q, L, cap, lookup, B)) + reserve


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("log_n", [16, 20, 23, 24])
def test_plan_falls_as_blocks_grow(bj, shape, log_n):
    plans = [_blocks_plan(bj, log_n, *SHAPES[shape], B) for B in (1, 2, 4, 8)]
    assert all(a >= b for a, b in zip(plans, plans[1:])), plans
    assert plans[1] < plans[0], plans  # the quotient's coset scratch is the peak at B = 1 on all three shapes


def test_production_shape_at_2p23_and_2p24(bj):
    """the quotient scratch (nat_cols() = 381 columns of n u64) sets the B = 1 peak of the production shape; cut into row blocks
    it stops doing so.  At 2^24 the plan and the natural-order inputs (155 variables and sigmas, 8 constants, 4 tables, the
    multiplicities) fit one 80 GB device together from B = 4 on, and not at B = 1."""
    p23 = [_blocks_plan(bj, 23, *SHAPES["production"], B) for B in (1, 2, 4, 8)]
    p24 = [_blocks_plan(bj, 24, *SHAPES["production"], B) for B in (1, 2, 4, 8)]
    assert p23[0] - p23[1] > 8 * GB
    inputs24 = 8 * (1 << 24) * (155 + 155 + 8 + 4 + 1)
    assert p24[0] + inputs24 > 80 * GB
    assert p24[2] + inputs24 < 80 * GB


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("B", [1, 2, 4, 8])
def test_lane_split_adds_up_to_the_plan(bj, shape, B):
    V, C, Q, L, cap, lookup = SHAPES[shape]
    one = bj.proof_memory_plan_lanes(20, V, C, Q, _cfg(L, cap), "recompute", 1, lookup=_lk(lookup), row_blocks=B)
    assert one["setup"] + one["lane"] == one["total"] == _blocks_plan(bj, 20, *SHAPES[shape], B)
    three = bj.proof_memory_plan_lanes(20, V, C, Q, _cfg(L, cap), "recompute", 3, lookup=_lk(lookup), row_blocks=B)
    assert three["setup"] == one["setup"] and three["lane"] == one["lane"] and three["total"] == one["setup"] + 3 * one["lane"]
    if B > 1:  # the setup's part is its trees alone, the same at any B; the lane's part falls with the quotient scratch
        base = bj.proof_memory_plan_lanes(20, V, C, Q, _cfg(L, cap), "recompute", 1, lookup=_lk(lookup))
        assert one["setup"] == base["setup"] and one["lane"] < base["lane"]


def test_invalid_block_counts_and_shapes_are_refused(bj):
    lib = bj.native.lib
    INVALID = bj.native.BJ_ERR_INVALID_ARG
    c = _circuit(bj, 10, 20, 6, 8, 2, 16, None)
    out = ctypes.c_uint64(7)
    for blocks in (0, 3, 5, 6, 16, 32):
        assert lib.bj_proof_memory_plan_recompute_blocks(ctypes.byref(c), blocks, ctypes.byref(out)) == INVALID and out.value == 0
    assert lib.bj_proof_memory_plan_recompute_blocks(ctypes.byref(c), 8, None) == INVALID
    assert lib.bj_proof_memory_plan_recompute_blocks(None, 2, ctypes.byref(out)) == INVALID
    # n / B >= 2 rows: log_n = 3 holds 4 blocks of 2 rows and not 8 of 1
    c = _circuit(bj, 3, 4, 2, 2, 2, 2, None)
    for blocks, status in ((1, 0), (2, 0), (4, 0), (8, INVALID)):
        assert lib.bj_proof_memory_plan_recompute_blocks(ctypes.byref(c), blocks, ctypes.byref(out)) == status, blocks
        assert (out.value > 0) == (status == 0)
    with pytest.raises(bj.BoojumError, match="bj_proof_memory_plan_recompute_blocks"):
        bj.proof_memory_plan_recompute_blocks(10, 20, 6, 8, _cfg(2, 16), 3)
    # row blocks belong to the recompute plan only
    c = _circuit(bj, 10, 20, 6, 8, 2, 16, None)
    lanes = (ctypes.c_uint64 * 3)()
    assert lib.bj_proof_memory_plan_lanes_host_blocks(ctypes.byref(c), bj.native.PLAN_RECOMPUTE, 4, 1, lanes) == 0 and lanes[2] > 0
    for plan in (bj.native.PLAN_RESIDENT, bj.native.PLAN_STREAMED):
        assert lib.bj_proof_memory_plan_lanes_host_blocks(ctypes.byref(c), plan, 2, 1, lanes) == INVALID
        assert lib.bj_proof_memory_plan_lanes_host_blocks(ctypes.byref(c), plan, 1, 1, lanes) == 0
    assert lib.bj_proof_memory_plan_lanes_host_blocks(ctypes.byref(c), bj.native.PLAN_RECOMPUTE, 3, 1, lanes) == INVALID
    # the switch needs a context; a context needs a device
    assert lib.bj_ctx_set_max_row_blocks(None, 2) == INVALID
    assert lib.bj_setup_row_blocks(None) == INVALID


def test_symbols_are_declared_and_exported(bj):
    import os
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "boojum_b200.h")).read()
    for name in ("bj_ctx_set_max_row_blocks", "bj_proof_memory_plan_recompute_blocks", "bj_setup_row_blocks",
                 "bj_proof_memory_plan_lanes_host_blocks"):
        assert "BJ_API int32_t %s(" % name in header, name
        assert hasattr(bj.native.lib, name), name
