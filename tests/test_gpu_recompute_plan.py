"""Proving on the recompute plan: one GPU, any quotient degree Q and LDE factor L, no coset of the setup, witness or stage-2
columns kept.  Their trees are built one committed coset at a time, the quotient evaluates every column it reads onto one
coset of [0, Q) at a time, and the openings, DEEP and the query answers rebuild the cosets they read from the natural-order
columns.  The plan is opt-in (Context.allow_recompute_plan); with it on, a limit between the recompute plan and the smallest
other plan makes bj_setup_create choose it.  The proof must not move: it is compared byte for byte with the resident proof of
the same inputs (and with the oracle's CPU prover on one shape), the verifier must accept it, and the context's pool must stay
at the planned peak.  With the switch off the same limit is refused exactly as before."""
import json
import threading

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


def _sha(bj, log_n, V, Q, lookup, pis):
    """the oracle's SHA-shaped circuit on the device; Q = 2 drops the gates (their degree needs Q = 4) and proves the copy
    permutation and lookup argument alone"""
    from era_boojum_b200 import synthetic
    from oracle import circuits
    c = circuits.sha_shaped(log_n, V, seed=400 + log_n, lookup=lookup)
    gates, oracle_gates = (synthetic.sha_shaped_gates(V), c["gates"]) if Q > 2 else ([], [])
    lk = None
    if lookup:
        lk = dict(c["lookup"], tables=bj.to_device(c["lookup"]["tables"]), multiplicities=bj.to_device(c["lookup"]["multiplicities"]))
    return dict(variables=bj.to_device(c["variables"]), sigmas=bj.to_device(c["sigmas"]), constants=bj.to_device(c["constants"]),
                gates=gates, oracle_gates=oracle_gates, lookup=lk, public_inputs=list(pis), cpu=c)


def _production(bj, log_n):
    """synthetic.generate_production_shaped: 155 columns, 11 gates, 8 lookups of width 3, 4 public inputs"""
    from era_boojum_b200 import synthetic
    ctx = bj.Context(0)
    c = synthetic.generate_production_shaped(ctx, log_n, seed=70 + log_n)
    ctx.synchronize()
    ctx.close()
    return c


def _plan(bj, log_n, c, Q, cfg, world=1):
    lk = c["lookup"]
    lk = dict(width=lk["width"], num_repetitions=lk["num_repetitions"]) if lk else None
    return bj.proof_memory_plan(log_n, c["sigmas"].shape[0], c["constants"].shape[0], Q, cfg, lookup=lk, world=world)


def _smallest_other(plan):
    return min(plan[k] for k in ("resident", "compact", "streamed") if plan[k])


def _setup(ctx, c, Q, cfg):
    return ctx.native_setup(c["sigmas"], c["constants"], c["gates"], Q, cfg, lookup=c["lookup"], public_inputs=c["public_inputs"])


def _prove(bj, c, Q, cfg, limit, allow):
    """setup + prove on a fresh context under `limit` (0: the device) -> (plan name, proof, setup cap, vk, pool high-water,
    memory_plan())"""
    ctx = bj.Context(0)
    ctx.set_memory_limit(limit)
    ctx.allow_recompute_plan(allow)
    try:
        nat = _setup(ctx, c, Q, cfg)
        m = c["lookup"]["multiplicities"] if c["lookup"] else None
        proof = nat.prove(c["variables"], m, as_json=True)
        out = (nat.plan, proof, nat.get_cap(), nat.vk(), ctx.memory_high_water(), nat.memory_plan())
        nat.close()
        ctx.synchronize()
        return out
    finally:
        ctx.close()


@pytest.mark.parametrize("shape,log_n,V,Q,L,cap,lookup,pis,hasher,transcript,pow_bits", [
    ("sha", 9, 20, 4, 8, 16, False, (), "poseidon2", "poseidon2", 0),                   # Q < L
    ("sha", 10, 20, 2, 4, 8, True, ((1, 3), (5, 3)), "blake2s", "blake2s", 0),         # Q < L
    ("sha", 10, 20, 4, 4, 8, True, ((2, 100),), "poseidon2", "poseidon", 0),           # Q = L: no other fallback
    ("sha", 11, 40, 8, 4, 16, True, ((0, 9),), "keccak256", "keccak256", 0),           # Q > L
    ("sha", 10, 20, 4, 8, 16, True, ((3, 5),), "poseidon2", "poseidon2", 10),          # proof of work
    ("production", 9, None, 8, 2, 32, True, None, "poseidon2", "poseidon2", 0),        # Q > L
    ("production", 10, None, 8, 2, 32, True, None, "blake2s", "blake2s", 0)])
def test_recompute_plan_proves_the_resident_proof_under_the_limit(bj, shape, log_n, V, Q, L, cap, lookup, pis, hasher, transcript, pow_bits):
    from era_boojum_b200 import prover
    c = _sha(bj, log_n, V, Q, lookup, pis) if shape == "sha" else _production(bj, log_n)
    cfg = prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100, pow_bits=pow_bits, hasher=hasher,
                             transcript=transcript)
    plan = _plan(bj, log_n, c, Q, cfg)
    assert plan["recompute"] is not None and plan["recompute"] < _smallest_other(plan)
    limit = (plan["recompute"] + _smallest_other(plan)) // 2

    kind, want, want_cap, _, high_resident, _ = _prove(bj, c, Q, cfg, 0, False)
    assert kind == "resident"
    kind, got, got_cap, vk, high, mp = _prove(bj, c, Q, cfg, limit, True)
    assert kind == "recompute"
    assert mp["pool"] + mp["outside_pool"] <= limit and mp["chunk"] >= 2
    # the pool's high-water mark on a fresh context is the planned pool peak, below the resident proof's
    assert high == mp["pool"], (high, mp)
    assert high < high_resident
    assert np.array_equal(got_cap, want_cap)
    assert got == want
    assert OV.verify(vk, json.loads(got))

    if shape == "sha" and log_n == 9:  # the oracle's CPU prover (Python integers)
        from oracle import prover as OP
        cpu = c["cpu"]
        ref, ref_cap = OP.prove(cpu["variables"], cpu["sigmas"], cpu["constants"], c["oracle_gates"], Q, L, cap, lookup=cpu["lookup"],
                                public_inputs=pis, hasher=hasher, transcript=transcript)
        assert np.array_equal(got_cap, ref_cap)
        assert json.dumps(json.loads(got), sort_keys=True) == json.dumps(ref, sort_keys=True)


def test_the_switch_off_keeps_the_refusal(bj):
    """the same limit without the switch: BJ_ERR_OOM before any launch, with the message of before (no recompute bytes)"""
    from era_boojum_b200 import prover
    c = _sha(bj, 10, 20, 4, True, ())
    cfg = prover.ProofConfig(fri_lde_factor=4, merkle_tree_cap_size=8, security_level=100)
    plan = _plan(bj, 10, c, 4, cfg)
    assert plan["compact"] is None and plan["streamed"] is None
    ctx = bj.Context(0)
    try:
        ctx.set_memory_limit((plan["recompute"] + plan["resident"]) // 2)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, 4, cfg)
        assert e.value.status == OOM
        msg = str(e.value)
        assert str(plan["resident"]) in msg and "recompute" not in msg and str(plan["recompute"]) not in msg
        assert ctx.launch_count() == before
    finally:
        ctx.close()


def test_limit_below_the_recompute_plan_is_refused(bj):
    from era_boojum_b200 import prover
    c = _production(bj, 10)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    plan = _plan(bj, 10, c, 8, cfg)
    ctx = bj.Context(0)
    try:
        ctx.allow_recompute_plan(True)
        ctx.set_memory_limit(plan["recompute"] - 1)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, 8, cfg)
        assert e.value.status == OOM
        msg = str(e.value)
        assert str(plan["resident"]) in msg and str(plan["streamed"]) in msg and str(plan["recompute"]) + " bytes on the recompute plan" in msg
        assert ctx.launch_count() == before
        # exactly at the recompute plan the setup is accepted, on the recompute plan
        ctx.set_memory_limit(plan["recompute"])
        nat = _setup(ctx, c, 8, cfg)
        assert nat.plan == "recompute" and not nat.compact
        nat.close()
    finally:
        ctx.close()


def test_a_sharded_context_ignores_the_switch(bj):
    """rank 0 of a 2-rank thread context, with the switch on, under a limit below its streamed plan: refused with BJ_ERR_OOM
    before the first collective (the other rank never joins), and the message names no recompute plan"""
    from era_boojum_b200 import prover
    c = _production(bj, 10)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    plan = _plan(bj, 10, c, 8, cfg, world=2)
    assert plan["recompute"] is None
    group = bj.Comm.local_group(2)
    ctx = bj.Context(0)
    comm = bj.Comm.local(ctx, group, 0, 2, 2)
    result = []

    def setup():
        try:
            result.append(_setup(ctx, c, 8, cfg))
        except bj.BoojumError as e:
            result.append(e)

    try:
        ctx.allow_recompute_plan(True)
        ctx.set_memory_limit(plan["streamed_sharded"] - 1)
        before = ctx.launch_count()
        t = threading.Thread(target=setup, daemon=True)
        t.start()
        t.join(timeout=120)
        assert not t.is_alive(), "bj_setup_create did not refuse before its first collective"
        e = result[0]
        assert isinstance(e, bj.BoojumError) and e.status == OOM
        assert str(plan["streamed_sharded"]) in str(e) and "recompute" not in str(e)
        assert ctx.launch_count() == before
    finally:
        comm.close()
        ctx.close()
        bj.Comm.destroy_local_group(group)


def test_prove_stream_on_the_recompute_plan(bj):
    """witness slots count the recompute plan plus the slot bytes; the streamed proofs are those of bj_prove one by one"""
    from era_boojum_b200 import prover, synthetic
    log_n = 10
    gen = bj.Context(0)
    cs = [synthetic.generate_production_shaped(gen, log_n, seed=95, witness_seed=700 + k) for k in range(3)]
    gen.synchronize()
    gen.close()
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    c0 = cs[0]
    plan = _plan(bj, log_n, c0, 8, cfg)
    V = c0["variables"].shape[0]
    slots_bytes = bj.witness_slots_bytes(log_n, V, 2, lookup=c0["lookup"])
    ctx = bj.Context(0)
    try:
        ctx.allow_recompute_plan(True)
        ctx.set_memory_limit(plan["recompute"] + 2 * slots_bytes)
        nat = _setup(ctx, c0, 8, cfg)
        assert nat.plan == "recompute"
        want = [nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in cs]
        assert len(set(want)) == len(want)
        hw = [(bj.to_numpy(c["variables"]), bj.to_numpy(c["lookup"]["multiplicities"])) for c in cs]
        slots = nat.witness_slots(2)
        assert list(nat.prove_stream(hw, slots=slots)) == want
        vk = nat.vk()
        assert all(OV.verify(vk, json.loads(p)) for p in want)
        slots.close()
        nat.close()
    finally:
        ctx.close()
