"""Proving under a device-memory limit when the quotient degree Q exceeds the LDE factor L (the production shape: Q = 8 over
L = 2).  A limit between the streamed and the resident plan makes bj_setup_create choose the streamed plan: the setup, witness
and stage-2 columns are evaluated on the committed cosets [0, L) only, and the quotient evaluates every column it reads onto
one coset of [L, Q) at a time.  The proof must not move: it is compared byte for byte with the resident proof of the same
inputs (and with the oracle's CPU prover on one shape), the verifier must accept it, and the context's pool must stay at the
planned peak.  A limit below the streamed plan is refused with BJ_ERR_OOM before any kernel runs."""
import json

import numpy as np
import pytest

from oracle import verifier as OV

pytestmark = pytest.mark.gpu

OOM = -4  # BJ_ERR_OOM


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


def _sha(bj, log_n, V, lookup, pis):
    """the oracle's SHA-shaped circuit (no specialised boolean gate), on the device"""
    from era_boojum_b200 import synthetic
    from oracle import circuits
    c = circuits.sha_shaped(log_n, V, seed=300 + log_n, lookup=lookup)
    lk = None
    if lookup:
        lk = dict(c["lookup"], tables=bj.to_device(c["lookup"]["tables"]), multiplicities=bj.to_device(c["lookup"]["multiplicities"]))
    return dict(variables=bj.to_device(c["variables"]), sigmas=bj.to_device(c["sigmas"]), constants=bj.to_device(c["constants"]),
                gates=synthetic.sha_shaped_gates(V), lookup=lk, public_inputs=list(pis), cpu=c)


def _production(bj, log_n):
    """synthetic.generate_production_shaped: 155 columns, 11 gates incl. the boolean gate on a specialised column, 8 lookups of
    width 3, 4 public inputs"""
    from era_boojum_b200 import synthetic
    ctx = bj.Context(0)
    c = synthetic.generate_production_shaped(ctx, log_n, seed=60 + log_n)
    ctx.synchronize()
    ctx.close()
    return c


def _plan(bj, log_n, c, Q, cfg):
    lk = c["lookup"]
    lk = dict(width=lk["width"], num_repetitions=lk["num_repetitions"]) if lk else None
    return bj.proof_memory_plan(log_n, c["sigmas"].shape[0], c["constants"].shape[0], Q, cfg, lookup=lk)


def _prove(bj, c, Q, cfg, limit):
    """setup + prove on a fresh context under `limit` (0: the device) -> (plan name, proof, setup cap, vk, pool high-water,
    memory_plan())"""
    ctx = bj.Context(0)
    ctx.set_memory_limit(limit)
    try:
        nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], Q, cfg, lookup=c["lookup"], public_inputs=c["public_inputs"])
        m = c["lookup"]["multiplicities"] if c["lookup"] else None
        proof = nat.prove(c["variables"], m, as_json=True)
        out = (nat.plan, proof, nat.get_cap(), nat.vk(), ctx.memory_high_water(), nat.memory_plan())
        assert nat.compact is False
        nat.close()
        ctx.synchronize()
        return out
    finally:
        ctx.close()


@pytest.mark.parametrize("shape,log_n,V,Q,L,cap,lookup,pis,hasher,transcript", [
    ("sha", 9, 20, 8, 2, 16, False, (), "poseidon2", "poseidon2"),
    ("sha", 10, 20, 4, 2, 8, True, ((1, 3), (5, 3)), "blake2s", "blake2s"),
    ("sha", 11, 40, 8, 4, 16, True, ((2, 100),), "poseidon2", "poseidon"),
    ("sha", 12, 20, 4, 2, 8, False, ((0, 9),), "keccak256", "keccak256"),
    ("production", 9, None, 8, 2, 32, True, None, "poseidon2", "poseidon2"),
    ("production", 10, None, 8, 4, 32, True, None, "blake2s", "blake2s"),
    ("production", 12, None, 8, 2, 32, True, None, "keccak256", "keccak256")])
def test_streamed_plan_proves_the_resident_proof_under_the_limit(bj, shape, log_n, V, Q, L, cap, lookup, pis, hasher, transcript):
    from era_boojum_b200 import prover
    c = _sha(bj, log_n, V, lookup, pis) if shape == "sha" else _production(bj, log_n)
    cfg = prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100, hasher=hasher, transcript=transcript)
    plan = _plan(bj, log_n, c, Q, cfg)
    assert plan["compact"] is None and plan["streamed"] is not None and plan["streamed"] < plan["resident"]
    limit = (plan["streamed"] + plan["resident"]) // 2

    kind, want, want_cap, _, high_resident, _ = _prove(bj, c, Q, cfg, 0)
    assert kind == "resident"
    kind, got, got_cap, vk, high, mp = _prove(bj, c, Q, cfg, limit)
    assert kind == "streamed"
    assert mp["pool"] + mp["outside_pool"] == plan["streamed"] <= limit and mp["chunk"] == 0
    # the pool's high-water mark on a fresh context is the planned pool peak, below the resident proof's
    assert high == mp["pool"], (high, mp)
    assert high < high_resident
    assert np.array_equal(got_cap, want_cap)
    assert got == want
    assert OV.verify(vk, json.loads(got))

    if shape == "sha" and log_n == 9:  # the oracle's CPU prover (Python integers)
        from oracle import prover as OP
        cpu = c["cpu"]
        ref, ref_cap = OP.prove(cpu["variables"], cpu["sigmas"], cpu["constants"], cpu["gates"], Q, L, cap, lookup=cpu["lookup"],
                                public_inputs=pis, hasher=hasher, transcript=transcript)
        assert np.array_equal(got_cap, ref_cap)
        assert json.dumps(json.loads(got), sort_keys=True) == json.dumps(ref, sort_keys=True)


def test_limit_below_the_streamed_plan_is_refused(bj):
    from era_boojum_b200 import prover
    c = _sha(bj, 10, 20, True, ())
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=8, security_level=100)
    plan = _plan(bj, 10, c, 8, cfg)
    ctx = bj.Context(0)
    ctx.set_memory_limit(plan["streamed"] - 1)
    before = ctx.launch_count()
    with pytest.raises(bj.BoojumError) as e:
        ctx.native_setup(c["sigmas"], c["constants"], c["gates"], 8, cfg, lookup=c["lookup"])
    assert e.value.status == OOM
    msg = str(e.value)
    assert "no compact plan" in msg and str(plan["resident"]) in msg and str(plan["streamed"]) in msg
    assert ctx.launch_count() == before
    # exactly at the streamed plan the setup is accepted, on the streamed plan
    ctx.set_memory_limit(plan["streamed"])
    nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], 8, cfg, lookup=c["lookup"])
    assert nat.plan == "streamed" and not nat.compact
    nat.close()
    ctx.close()
