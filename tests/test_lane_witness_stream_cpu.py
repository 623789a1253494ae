"""Witness slot sets on proof lanes without a GPU: bj_witness_slots_bytes_split against the slot set's pool allocations listed
one by one (what a set allocates in its own context's pool, and the u32 variables hint that lives once on the setup), its sum
against bj_witness_slots_bytes, its refusals, and its declaration and export."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCTION_LOOKUP = dict(width=3, num_repetitions=8)


@pytest.fixture(scope="module")
def bj():
    import era_boojum_b200 as m
    return m


def _pool(n_u64):
    return 8 * max(n_u64, 1)


def _own_allocations(log_n, V, n_slots, max_values, lookup):
    """the pool allocations bj_witness_slots_create makes in the set's own context (u64 counts)"""
    n, lk = 1 << log_n, 1 if lookup else 0
    out = [n_slots * (V + lk) * n]
    if max_values:
        out.append(max_values)
        if lookup:
            out.append((n + 1) // 2)
    return out


@pytest.mark.parametrize("lookup", [None, dict(width=3, num_repetitions=8)])
@pytest.mark.parametrize("max_values", [0, 1, 12345, 1 << 22])
@pytest.mark.parametrize("n_slots", [1, 2, 3, 4])
def test_split_adds_up_to_the_slot_bytes(bj, lookup, max_values, n_slots):
    for log_n, V in ((1, 1), (10, 20), (16, 60), (20, 155), (21, 92)):
        own, hint = bj.witness_slots_bytes_split(log_n, V, n_slots, max_values, lookup=lookup)
        assert own == sum(_pool(a) for a in _own_allocations(log_n, V, n_slots, max_values, lookup)), (log_n, V)
        # the hint: ceil(V * n / 2) u64 (V * n u32) when the set takes WitnessVecs, else nothing
        assert hint == (_pool((V * (1 << log_n) + 1) // 2) if max_values else 0), (log_n, V)
        assert own + hint == bj.witness_slots_bytes(log_n, V, n_slots, max_values, lookup=lookup, world=1)


def test_split_of_the_production_shape(bj):
    # 2^20 rows, 155 columns + multiplicities: a lane's 2-slot WitnessVec set holds two slots, all_values and n u32
    # multiplicities; the 155 * 2^20 u32 hint is the setup's
    own, hint = bj.witness_slots_bytes_split(20, 155, 2, 155 << 20, lookup=PRODUCTION_LOOKUP)
    assert own == 2 * (156 * 8 << 20) + (155 << 23) + (1 << 22)
    assert hint == 155 << 22
    assert bj.witness_slots_bytes_split(20, 155, 2, 0, lookup=PRODUCTION_LOOKUP) == (2 * (156 * 8 << 20), 0)


@pytest.mark.parametrize("log_n,V,n_slots", [(10, 20, 0), (10, 20, 5), (0, 20, 1), (29, 20, 1), (10, 0, 1)])
def test_split_refuses_bad_shapes(bj, log_n, V, n_slots):
    with pytest.raises(bj.BoojumError) as e:
        bj.witness_slots_bytes_split(log_n, V, n_slots, 0)
    assert e.value.status == bj.native.BJ_ERR_INVALID_ARG


def test_split_refuses_null_pointers(bj):
    lib = bj.native.lib
    c = bj.native.Circuit()
    c.log_n, c.num_variables = 10, 20
    out = (ctypes.c_uint64 * 2)(7, 7)
    assert lib.bj_witness_slots_bytes_split(None, 2, 0, out) == bj.native.BJ_ERR_INVALID_ARG
    assert lib.bj_witness_slots_bytes_split(ctypes.byref(c), 2, 0, None) == bj.native.BJ_ERR_INVALID_ARG
    assert list(out) == [7, 7]
    assert lib.bj_witness_slots_bytes_split(ctypes.byref(c), 2, 0, out) == bj.native.BJ_OK and out[1] == 0


def test_lane_slot_sets_need_a_device(bj):
    """with no device there is no context: creating a set on a NULL context is refused before anything else"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = ctypes.c_void_p()
    assert bj.native.lib.bj_witness_slots_create(None, None, 2, 0, ctypes.byref(h)) == bj.native.BJ_ERR_INVALID_ARG
    assert not h.value


def test_split_is_declared_and_exported(bj):
    hdr = open(os.path.join(ROOT, "include", "boojum_b200.h")).read()
    declared = set(re.findall(r"BJ_API\s+[\w\s\*]+?\b(bj_\w+)\s*\(", hdr))
    assert "bj_witness_slots_bytes_split" in declared and "bj_witness_slots_bytes_split" in bj.native.SIGNATURES
    assert hasattr(bj.native.lib, "bj_witness_slots_bytes_split")
    assert hasattr(bj, "witness_slots_bytes_split")
    import inspect
    assert "ctx" in inspect.signature(bj.NativeSetup.witness_slots).parameters
    assert "ctx" in inspect.signature(bj.WitnessSlots).parameters
    assert "slots_per_lane" in inspect.signature(bj.NativeSetup.prove_concurrent).parameters
