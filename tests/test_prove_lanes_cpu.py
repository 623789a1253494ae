"""bj_proof_memory_plan_lanes_host (no GPU): the device bytes of one setup proved on N lanes at once, counted from the circuit's
shapes.  Every plan splits into the setup's part (the pool bytes the setup keeps and the twiddle / coset-power tables the lanes
share) and one lane's part (what a proof's pool adds on top of the setup, and the lane's own scratch and parameter arena).  At
one lane the two add up to the single-context plan; each further lane adds its part once."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANS = ("resident", "compact", "streamed", "recompute")


@pytest.fixture(scope="module")
def bj():
    import era_boojum_b200 as m
    return m


def _cfg(L, cap):
    from era_boojum_b200 import prover
    return prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100)


def _lanes(bj, log_n, V, C, Q, L, cap, lookup, plan, n_lanes):
    lk = dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None
    return bj.proof_memory_plan_lanes(log_n, V, C, Q, _cfg(L, cap), plan, n_lanes, lookup=lk)


def _plan(bj, log_n, V, C, Q, L, cap, lookup):
    lk = dict(width=lookup[0], num_repetitions=lookup[1]) if lookup else None
    return bj.proof_memory_plan(log_n, V, C, Q, _cfg(L, cap), lookup=lk)


def _circuit(bj, log_n, V, C, Q, L, cap, lookup):
    c = bj.native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree, c.fri_lde_factor, c.merkle_tree_cap_size = log_n, V, C, Q, L, cap
    c.security_level = 100
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup
    return c


# (log_n, V, C, Q, L, cap, lookup): the production shape (Q > L), the bench shape (Q < L), a Q = L shape, small shapes
SHAPES = [(20, 155, 8, 8, 2, 32, (3, 8)), (16, 92, 7, 4, 8, 16, (4, 8)), (21, 92, 7, 4, 8, 16, (4, 8)), (18, 92, 7, 4, 4, 16, (4, 8)),
          (10, 20, 6, 2, 4, 8, (4, 2)), (12, 40, 6, 4, 8, 16, None), (11, 20, 6, 8, 2, 16, None)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("plan", PLANS)
def test_one_lane_is_the_plan(bj, shape, plan):
    want = _plan(bj, *shape)[plan]
    got = _lanes(bj, *shape, plan, 1)
    if want is None:
        assert got is None
        return
    assert got["setup"] > 0 and got["lane"] > 0
    assert got["setup"] + got["lane"] == got["total"] == want


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("plan", PLANS)
def test_each_lane_adds_its_part(bj, shape, plan):
    first = _lanes(bj, *shape, plan, 1)
    if first is None:
        return
    totals = []
    for n in range(1, 9):
        got = _lanes(bj, *shape, plan, n)
        assert (got["setup"], got["lane"]) == (first["setup"], first["lane"])
        assert got["total"] == got["setup"] + n * got["lane"]
        totals.append(got["total"])
    assert all(a < b for a, b in zip(totals, totals[1:]))


def test_resident_setup_part_is_the_setup_lde_tree_and_tables(bj):
    """the resident setup keeps its LDE on all D = max(L, Q) cosets and its tree; the lanes share the twiddles of the
    factor-D domain and the coset-power tables (capped by their 3 GiB budget)"""
    log_n, V, C, Q, L, cap, lookup = 16, 92, 7, 4, 8, 16, (4, 8)
    n, D, S = 1 << log_n, max(L, Q), V + C + lookup[0] + 1
    log_d = D.bit_length() - 1
    tables = 8 * n * D + min(3 << 30, 8 * n * (D + Q + 2)) + 64 * 16 * (1 << ((log_n + log_d + 2) // 2))
    setup_pool = 8 * (S * n * D + 4 * n * L + 4 * (n * L - cap))
    got = _lanes(bj, log_n, V, C, Q, L, cap, lookup, "resident", 1)
    assert got["setup"] == setup_pool + tables
    # the lane keeps no setup column and no shared table: its part is the proof's pool plus its scratch and arena
    assert got["lane"] == got["total"] - got["setup"]
    assert got["lane"] - (8 * max(1 << 27, 4 * n) + (16 << 20)) < got["total"] - setup_pool - tables


def test_lanes_of_the_production_shape_share_most_of_the_memory(bj):
    """the production shape at 2^20 rows: the setup's part is a large share of the plan, so a second lane costs less than a
    second context with its own setup"""
    shape = (20, 155, 8, 8, 2, 32, (3, 8))
    one = _lanes(bj, *shape, "resident", 1)
    two = _lanes(bj, *shape, "resident", 2)
    assert two["total"] < 2 * one["total"]
    assert one["setup"] > 0.3 * one["total"]


def test_invalid_arguments_are_refused(bj):
    lib = bj.native.lib
    out = (ctypes.c_uint64 * 3)()
    c = _circuit(bj, 12, 20, 6, 4, 8, 16, None)
    assert lib.bj_proof_memory_plan_lanes_host(ctypes.byref(c), 0, 1, out) == 0 and out[2] > 0
    assert lib.bj_proof_memory_plan_lanes_host(ctypes.byref(c), 0, 0, out) == bj.native.BJ_ERR_INVALID_ARG   # no lane
    assert lib.bj_proof_memory_plan_lanes_host(ctypes.byref(c), 4, 1, out) == bj.native.BJ_ERR_INVALID_ARG   # no such plan
    assert lib.bj_proof_memory_plan_lanes_host(None, 0, 1, out) == bj.native.BJ_ERR_INVALID_ARG
    assert lib.bj_proof_memory_plan_lanes_host(ctypes.byref(c), 0, 1, None) == bj.native.BJ_ERR_INVALID_ARG
    c.quotient_degree = 3
    assert lib.bj_proof_memory_plan_lanes_host(ctypes.byref(c), 0, 1, out) == bj.native.BJ_ERR_INVALID_ARG   # Q not a power of two
    assert lib.bj_proof_memory_plan_lanes(None, 1, out) == bj.native.BJ_ERR_INVALID_ARG
    assert lib.bj_proof_memory_plan_lane_pool(None, out) == bj.native.BJ_ERR_INVALID_ARG
    with pytest.raises(bj.BoojumError, match="bj_proof_memory_plan_lanes_host"):
        _lanes(bj, 12, 20, 6, 4, 8, 16, None, "resident", 0)
    with pytest.raises(KeyError):
        _lanes(bj, 12, 20, 6, 4, 8, 16, None, "sharded", 1)
    # a plan that does not apply to the circuit: zeros, None in Python
    c.quotient_degree = 8
    assert lib.bj_proof_memory_plan_lanes_host(ctypes.byref(c), 1, 1, out) == 0 and list(out) == [0, 0, 0]   # compact needs Q < L
    assert _lanes(bj, 12, 20, 6, 8, 8, 16, None, "streamed", 2) is None                                       # streamed needs Q > L


def test_lane_symbols_are_declared_and_exported(bj):
    hdr = open(os.path.join(ROOT, "include", "boojum_b200.h")).read()
    declared = set(re.findall(r"BJ_API\s+[\w\s\*]+?\b(bj_\w+)\s*\(", hdr))
    for name in ("bj_ctx_create_lane", "bj_proof_memory_plan_lanes", "bj_proof_memory_plan_lanes_host", "bj_proof_memory_plan_lane_pool"):
        assert name in declared and name in bj.native.SIGNATURES
        assert hasattr(bj.native.lib, name)
    assert hasattr(bj.Context, "lane")
    assert hasattr(bj.NativeSetup, "prove_concurrent") and hasattr(bj.NativeSetup, "memory_plan_lanes")


def test_no_lane_without_a_device(bj):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = ctypes.c_void_p()
    assert bj.native.lib.bj_ctx_create_lane(None, ctypes.byref(h)) == bj.native.BJ_ERR_INVALID_ARG
    assert bj.native.lib.bj_ctx_create_lane(None, None) == bj.native.BJ_ERR_INVALID_ARG
