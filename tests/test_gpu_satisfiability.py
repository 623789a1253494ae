"""bj_check_satisfied / bj_lookup_multiplicities on the GPU: the device report equals, field for field, the oracle's
(oracle/satisfiability.py) and the report written down from each mutation's construction (the catalogue of
tests/test_satisfiability_cpu.py); reports agree with what bj_prove does with the same inputs; the device multiplicity column
equals the circuit's and proves bit-identically; misuse is refused before any launch."""
import json

import numpy as np
import pytest

from oracle import satisfiability as OS
from oracle import verifier as OV
from oracle.gates import P
from tests import test_satisfiability_cpu as CAT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    import era_boojum_b200 as bj
    from era_boojum_b200 import prover, synthetic
    ctx = bj.Context.on_current_stream(0)
    yield bj, ctx, prover, synthetic
    ctx.synchronize()
    ctx.close()


def _device(bj, c):
    lk = None
    if c["lookup"]:
        lk = dict(c["lookup"], tables=bj.to_device(c["lookup"]["tables"]), multiplicities=bj.to_device(c["lookup"]["multiplicities"]))
    return bj.to_device(c["variables"]), bj.to_device(c["sigmas"]), bj.to_device(c["constants"]), lk


def device_report(env, c, ctx=None):
    bj, ctx0, _, _ = env
    v, s, k, lk = _device(bj, c)
    return (ctx or ctx0).check_if_satisfied(v, s, k, c["gates"], lookup=lk)


def _circuit(kind, log_n):
    return CAT.sha_circuit(log_n) if kind == "sha" else CAT.production_circuit(log_n)


SHAPES = [("sha", 5), ("sha", 10), ("sha", 12), ("production", 5), ("production", 10)]


@pytest.mark.parametrize("kind,log_n", SHAPES)
def test_satisfied_circuits_report_nothing(env, kind, log_n):
    c = _circuit(kind, log_n)
    assert device_report(env, c) == CAT.expect()


@pytest.mark.parametrize("log_n,V,lookup", [(6, 20, False), (7, 40, True), (8, 40, False)])
def test_satisfied_sha_variants(env, log_n, V, lookup):
    c = CAT.sha_circuit(log_n, seed=log_n, V=V, lookup=lookup)
    assert device_report(env, c) == CAT.oracle_report(c) == CAT.expect()


@pytest.mark.parametrize("log_n", [5, 10, 12])
@pytest.mark.parametrize("mutation", CAT.SHA_MUTATIONS, ids=lambda m: m.__name__)
def test_mutations_sha(env, mutation, log_n):
    m, want = CAT.mutated(CAT.sha_circuit(log_n), mutation)
    got = device_report(env, m)
    assert got == want
    if log_n <= 10:
        assert got == CAT.oracle_report(m)


@pytest.mark.parametrize("log_n", [5, 10])
@pytest.mark.parametrize("mutation", CAT.PRODUCTION_MUTATIONS, ids=lambda m: m.__name__)
def test_mutations_production(env, mutation, log_n):
    m, want = CAT.mutated(CAT.production_circuit(log_n), mutation)
    got = device_report(env, m)
    assert got == want
    if log_n <= 5:
        assert got == CAT.oracle_report(m)


@pytest.mark.parametrize("log_n", [11, 12])
def test_padding_multiplicity(env, log_n):
    m, want = CAT.mutated(CAT.sha_circuit(log_n), CAT.padding_multiplicity)
    assert device_report(env, m) == want


def _non_canonical(a):
    """x + p wherever that fits in 64 bits"""
    a = a.copy()
    small = a < np.uint64(2 ** 64 - P)
    a[small] += np.uint64(P)
    return a


@pytest.mark.parametrize("kind,log_n", [("sha", 10), ("production", 6)])
def test_non_canonical_inputs_are_not_failures(env, kind, log_n):
    c = _circuit(kind, log_n)
    nc = dict(c, variables=_non_canonical(c["variables"]), sigmas=_non_canonical(c["sigmas"]), constants=_non_canonical(c["constants"]))
    nc["lookup"] = dict(c["lookup"], tables=_non_canonical(c["lookup"]["tables"]), multiplicities=_non_canonical(c["lookup"]["multiplicities"]))
    assert not np.array_equal(nc["variables"], c["variables"])
    assert device_report(env, nc) == CAT.expect()


def test_same_report_on_a_sharded_context(env):
    bj = env[0]
    m, want = CAT.mutated(CAT.sha_circuit(10), CAT.several)
    other = bj.Context.on_current_stream(0)
    try:
        other.set_domain_shard(1, 4, 2)
        assert device_report(env, m, ctx=other) == want == device_report(env, m)
    finally:
        other.close()


# ---- reports agree with the prover ----
def _prove(env, c, L=4, cap=8, multiplicities=None):
    bj, ctx, prover, _ = env
    v, s, k, lk = _device(bj, c)
    cfg = prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100)
    nat = ctx.native_setup(s, k, c["gates"], c["quotient_degree"], cfg, lookup=lk)
    try:
        m = multiplicities if multiplicities is not None else (lk["multiplicities"] if lk else None)
        return nat.vk(), nat.prove(v, m)
    finally:
        nat.close()


def test_satisfied_circuits_prove(env):
    for c in (CAT.sha_circuit(6), CAT.production_circuit(5)):
        assert device_report(env, c)["satisfied"] == 1
        vk, proof = _prove(env, c, L=2 if c["quotient_degree"] == 8 else 4, cap=4)
        assert proof["values_at_z"]


@pytest.mark.parametrize("mutation", CAT.SHA_MUTATIONS + CAT.PRODUCTION_MUTATIONS, ids=lambda m: m.__name__)
def test_mutated_circuits_are_refused_by_the_prover(env, mutation):
    """a gate, copy or sigma failure makes bj_prove return BJ_ERR_INVALID_ARG; a lookup failure alone (bj_prove does not
    check the log-derivative sum) yields a proof that the verifier rejects"""
    bj = env[0]
    prod = mutation in CAT.PRODUCTION_MUTATIONS
    m, want = CAT.mutated(CAT.production_circuit(5) if prod else CAT.sha_circuit(6), mutation)
    assert device_report(env, m) == want
    L, cap = (2, 4) if prod else (4, 8)
    if want["gate_failures"] or want["copy_failures"] or want["sigma_failures"]:
        with pytest.raises(bj.BoojumError) as e:
            _prove(env, m, L, cap)
        assert e.value.status == bj.native.BJ_ERR_INVALID_ARG
    else:
        vk, proof = _prove(env, m, L, cap)
        with pytest.raises(AssertionError):
            OV.verify(vk, proof)


# ---- bj_lookup_multiplicities ----
@pytest.mark.parametrize("log_n", [8, 11, 14])
def test_device_multiplicities_equal_the_circuit_column(env, log_n):
    bj, ctx, _, synthetic = env
    variables, sigmas, constants, gates, Q, lk = synthetic.generate(ctx, log_n, 60, seed=log_n, lookup=True)
    got = ctx.materialize_multiplicities_polynomials(variables, constants, lk)
    assert bj.to_numpy(got).tolist() == bj.to_numpy(lk["multiplicities"]).tolist()


def test_device_multiplicities_production_shape(env):
    bj, ctx, _, synthetic = env
    c = synthetic.generate_production_shaped(ctx, 12, seed=4)
    got = ctx.materialize_multiplicities_polynomials(c["variables"], c["constants"], c["lookup"])
    assert bj.to_numpy(got).tolist() == bj.to_numpy(c["lookup"]["multiplicities"]).tolist()


def test_device_multiplicities_match_the_oracle_and_prove_identically(env):
    bj, ctx, _, _ = env
    c = CAT.sha_circuit(11)
    v, s, k, lk = _device(bj, c)
    got = ctx.materialize_multiplicities_polynomials(v, k, lk)
    assert bj.to_numpy(got).tolist() == OS.multiplicities(c["variables"], c["constants"], c["lookup"])
    _, want = _prove(env, c)
    _, proof = _prove(env, c, multiplicities=got)
    assert json.dumps(proof, sort_keys=True) == json.dumps(want, sort_keys=True)


def test_device_multiplicities_refuse_an_unmatched_tuple(env):
    bj, ctx, _, _ = env
    m, _ = CAT.mutated(CAT.sha_circuit(8), CAT.lookup_off_table)
    v, s, k, lk = _device(bj, m)
    with pytest.raises(bj.BoojumError) as e:
        ctx.materialize_multiplicities_polynomials(v, k, lk)
    assert e.value.status == bj.native.BJ_ERR_INVALID_ARG and "row 255" in str(e.value)


# ---- at scale: the benchmark circuits ----
@pytest.mark.parametrize("shape", ["sha22", "production20"])
def test_bench_circuits_at_scale(env, shape):
    bj, ctx, _, synthetic = env
    torch = ctx._torch
    if shape == "sha22":
        variables, sigmas, constants, gates, Q, lk = synthetic.generate(ctx, 22, 60, seed=42, lookup=True)
    else:
        c = synthetic.generate_production_shaped(ctx, 20, seed=0)
        variables, sigmas, constants, gates, lk = c["variables"], c["sigmas"], c["constants"], c["gates"], c["lookup"]
    assert ctx.check_if_satisfied(variables, sigmas, constants, gates, lookup=lk) == CAT.expect()
    # one mutation in the last row: SHA shape - cell (0, r) + 1, read by the gate every row kind selects and tied to nothing
    # (its report comes from the oracle on that row); production shape - the boolean gate's column set to 2
    n = variables.shape[1]
    r = n - 1
    bad = variables.clone()
    if shape == "sha22":
        bad[0, r] += 1
        row = OS.empty_report()
        OS.check_gates(bj.to_numpy(bad[:, r:r + 1]), bj.to_numpy(constants[:, r:r + 1]),
                       [(g["name"], g["num_repetitions"], g["selector_path"]) for g in gates], row)
        assert row["gate_failures"]
        want = OS.finish(dict(row, gate_row=r))
    else:
        bad[154, r] = 2
        want = CAT.expect(gate_failures=1, gate_row=r, gate_index=0, gate_repetition=0, gate_term=0, gate_value=P - 2, gate_selector=1)
    assert ctx.check_if_satisfied(bad, sigmas, constants, gates, lookup=lk) == want
    del bad
    torch.cuda.empty_cache()


# ---- misuse ----
def test_misuse_is_refused_without_a_launch(env):
    bj, ctx, _, _ = env
    import ctypes
    N = bj.native
    c = CAT.sha_circuit(6)
    v, s, k, lk = _device(bj, c)
    circ, keep = bj._circuit(ctx, 6, v.shape[0], k.shape[0], c["gates"], lk)
    rep = N.SatisfiabilityReport()
    P_ = ctx._ptr

    def call(circuit=circ, sig=P_(s), con=P_(k), tab=P_(lk["tables"]), var=P_(v), mult=P_(lk["multiplicities"])):
        return N.lib.bj_check_satisfied(ctx._h, ctypes.byref(circuit), sig, con, tab, var, mult, ctypes.byref(rep))

    ctx.synchronize()
    before = ctx.launch_count()
    cases = [dict(sig=None), dict(var=None), dict(con=None), dict(tab=None), dict(mult=None)]
    for case in cases:
        assert call(**case) == N.BJ_ERR_INVALID_ARG, case
        assert N.lib.bj_last_error(ctx._h).decode()
    bad = N.Circuit.from_buffer_copy(circ)
    bad.lookup_table_id_column = k.shape[0]
    assert call(circuit=bad) == N.BJ_ERR_INVALID_ARG and "table-id" in N.lib.bj_last_error(ctx._h).decode()
    gates = [dict(g) for g in c["gates"]]
    gates[1] = dict(gates[1], relations=[(N.REL_MUL, 0, (N.IDX_VARIABLE, 500), (N.IDX_VARIABLE, 1))], writes=[(N.IDX_TEMPORARY, 0)])
    badg, keep2 = bj._circuit(ctx, 6, v.shape[0], k.shape[0], gates, lk)
    assert call(circuit=badg) == N.BJ_ERR_INVALID_ARG and "gate program" in N.lib.bj_last_error(ctx._h).decode()
    m = bj.to_device(np.zeros(64, np.uint64))
    assert N.lib.bj_lookup_multiplicities(ctx._h, ctypes.byref(circ), P_(k), None, P_(v), P_(m)) == N.BJ_ERR_INVALID_ARG
    nolk, keep3 = bj._circuit(ctx, 6, v.shape[0], k.shape[0], c["gates"], None)
    assert N.lib.bj_lookup_multiplicities(ctx._h, ctypes.byref(nolk), P_(k), P_(lk["tables"]), P_(v), P_(m)) == N.BJ_ERR_INVALID_ARG
    assert ctx.launch_count() == before
    assert call() == N.BJ_OK and rep.satisfied == 1
