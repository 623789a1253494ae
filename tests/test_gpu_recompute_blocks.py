"""Proving on the one-GPU recompute plan with every coset cut into B row blocks (Context.set_max_row_blocks).  The trees are
built one row block of n / B rows at a time and the quotient evaluates every column it reads, and z(omega x), onto one of the
Q * B row blocks of cosets [0, Q) at a time; the openings, DEEP and the query answers rebuild whole cosets as on the recompute
plan.  The proof must not move: for B = 2, 4 and 8 it is compared byte for byte with the resident proof of the same inputs, the
verifier must accept it, and the context's pool must stay at the planned peak.  A limit picks the fewest row blocks that fit,
the refusal below every plan names the bytes at the most row blocks allowed, and with the default switch (one block) every
choice and refusal is the recompute plan's of before."""
import json

import numpy as np
import pytest

from oracle import verifier as OV

pytestmark = pytest.mark.gpu

OOM, INVALID = -4, -1  # BJ_ERR_OOM, BJ_ERR_INVALID_ARG


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


def _sha(bj, log_n, V, Q, lookup, pis):
    """the oracle's SHA-shaped circuit on the device; Q = 2 drops the gates (their degree needs Q = 4)"""
    from era_boojum_b200 import synthetic
    from oracle import circuits
    c = circuits.sha_shaped(log_n, V, seed=500 + log_n, lookup=lookup)
    gates = synthetic.sha_shaped_gates(V) if Q > 2 else []
    lk = None
    if lookup:
        lk = dict(c["lookup"], tables=bj.to_device(c["lookup"]["tables"]), multiplicities=bj.to_device(c["lookup"]["multiplicities"]))
    return dict(variables=bj.to_device(c["variables"]), sigmas=bj.to_device(c["sigmas"]), constants=bj.to_device(c["constants"]),
                gates=gates, lookup=lk, public_inputs=list(pis))


def _production(bj, log_n, witness_seeds=(None,)):
    """synthetic.generate_production_shaped: 155 columns, 11 gates, 8 lookups of width 3, 4 public inputs"""
    from era_boojum_b200 import synthetic
    ctx = bj.Context(0)
    kw = lambda ws: {} if ws is None else {"witness_seed": ws}
    cs = [synthetic.generate_production_shaped(ctx, log_n, seed=80 + log_n, **kw(ws)) for ws in witness_seeds]
    ctx.synchronize()
    ctx.close()
    return cs


def _lk(c):
    lk = c["lookup"]
    return dict(width=lk["width"], num_repetitions=lk["num_repetitions"]) if lk else None


def _plan(bj, log_n, c, Q, cfg):
    return bj.proof_memory_plan(log_n, c["sigmas"].shape[0], c["constants"].shape[0], Q, cfg, lookup=_lk(c))


def _blocks(bj, log_n, c, Q, cfg, B):
    return bj.proof_memory_plan_recompute_blocks(log_n, c["sigmas"].shape[0], c["constants"].shape[0], Q, cfg, B, lookup=_lk(c))


def _setup(ctx, c, Q, cfg):
    return ctx.native_setup(c["sigmas"], c["constants"], c["gates"], Q, cfg, lookup=c["lookup"], public_inputs=c["public_inputs"])


def _mult(c):
    return c["lookup"]["multiplicities"] if c["lookup"] else None


def _prove(bj, c, Q, cfg, limit, allow, max_blocks=1):
    """setup + prove on a fresh context -> (plan name, row blocks, proof, setup cap, vk, pool high-water, memory_plan())"""
    ctx = bj.Context(0)
    ctx.set_memory_limit(limit)
    ctx.allow_recompute_plan(allow)
    ctx.set_max_row_blocks(max_blocks)
    try:
        nat = _setup(ctx, c, Q, cfg)
        proof = nat.prove(c["variables"], _mult(c), as_json=True)
        out = (nat.plan, nat.row_blocks, proof, nat.get_cap(), nat.vk(), ctx.memory_high_water(), nat.memory_plan())
        nat.close()
        ctx.synchronize()
        return out
    finally:
        ctx.close()


def _cfg(L, cap, hasher="poseidon2", transcript="poseidon2"):
    from era_boojum_b200 import prover
    return prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100, hasher=hasher, transcript=transcript)


@pytest.mark.parametrize("shape,log_n,V,Q,L,cap,lookup,pis,hasher,transcript", [
    # wide circuits: at 2^10 rows the quotient's unit scratch sets the pool peak up to B = 8, so each B is the fewest that fit
    ("sha", 10, 80, 2, 4, 8, False, ((1, 3), (5, 3)), "poseidon2", "poseidon2"),     # Q < L (Q = 2: no gates)
    ("sha", 10, 80, 2, 4, 8, True, ((2, 100),), "blake2s", "blake2s"),              # Q < L
    ("sha", 10, 120, 4, 4, 8, True, ((0, 9),), "keccak256", "keccak256"),           # Q = L
    ("sha", 10, 200, 8, 4, 16, False, (), "poseidon2", "poseidon"),                 # Q > L
    ("production", 10, None, 8, 2, 32, True, None, "poseidon2", "poseidon2"),       # Q > L, the production shape
    ("production", 13, None, 8, 2, 32, True, None, "blake2s", "blake2s")])
def test_row_blocks_prove_the_resident_proof(bj, shape, log_n, V, Q, L, cap, lookup, pis, hasher, transcript):
    c = _sha(bj, log_n, V, Q, lookup, pis) if shape == "sha" else _production(bj, log_n)[0]
    cfg = _cfg(L, cap, hasher, transcript)
    plans = {B: _blocks(bj, log_n, c, Q, cfg, B) for B in (1, 2, 4, 8)}
    assert plans[1] > plans[2] > plans[4] > plans[8], plans
    kind, _, want, want_cap, _, _, _ = _prove(bj, c, Q, cfg, 0, False)
    assert kind == "resident"
    for B in (2, 4, 8):
        # the limit of B's own plan, with up to 8 row blocks allowed: the fewest that fit are B
        kind, blocks, got, got_cap, vk, high, mp = _prove(bj, c, Q, cfg, plans[B], True, 8)
        assert (kind, blocks) == ("recompute", B)
        assert mp["pool"] + mp["outside_pool"] <= plans[B] and mp["chunk"] >= 2
        assert high == mp["pool"], (B, high, mp)
        assert np.array_equal(got_cap, want_cap), B
        assert got == want, B
    assert OV.verify(vk, json.loads(got))


def _production_case(bj):
    c = _production(bj, 11)[0]
    cfg = _cfg(2, 32)
    return c, cfg, _plan(bj, 11, c, 8, cfg), {B: _blocks(bj, 11, c, 8, cfg, B) for B in (1, 2, 4, 8)}


def test_the_fewest_row_blocks_that_fit_are_taken(bj):
    c, cfg, plan, blocks = _production_case(bj)
    assert blocks[1] == plan["recompute"] and blocks[2] < blocks[1]
    ctx = bj.Context(0)
    try:
        ctx.allow_recompute_plan(True)
        ctx.set_max_row_blocks(8)
        for limit, want in (((blocks[1] + blocks[2]) // 2, 2), (blocks[1], 1), ((plan["streamed"] + blocks[1]) // 2, 1),
                            (plan["streamed"], None)):
            ctx.set_memory_limit(limit)
            nat = _setup(ctx, c, 8, cfg)
            if want is None:
                assert nat.plan == "streamed" and nat.row_blocks == 1
            else:
                assert nat.plan == "recompute" and nat.row_blocks == want, (limit, nat.row_blocks)
                assert sum(nat.memory_plan()[k] for k in ("pool", "outside_pool")) == blocks[want]
            nat.close()
        # at most 4 allowed: a limit between the plans at 8 and 4 row blocks is refused, naming the plan at 4
        ctx.set_max_row_blocks(4)
        ctx.set_memory_limit((blocks[4] + blocks[8]) // 2)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, 8, cfg)
        assert e.value.status == OOM and str(blocks[4]) + " bytes on the recompute plan" in str(e.value)
        assert ctx.launch_count() == before
    finally:
        ctx.close()


def test_a_limit_below_the_plan_at_the_most_row_blocks_is_refused(bj):
    c, cfg, plan, blocks = _production_case(bj)
    ctx = bj.Context(0)
    try:
        ctx.allow_recompute_plan(True)
        ctx.set_max_row_blocks(8)
        ctx.set_memory_limit(blocks[8] - 1)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, 8, cfg)
        assert e.value.status == OOM
        msg = str(e.value)
        assert str(plan["resident"]) in msg and str(plan["streamed"]) in msg and str(blocks[8]) + " bytes on the recompute plan" in msg
        assert ctx.launch_count() == before
        ctx.set_memory_limit(blocks[8])
        nat = _setup(ctx, c, 8, cfg)
        assert nat.plan == "recompute" and nat.row_blocks == 8
        nat.close()
    finally:
        ctx.close()


def test_the_default_switch_keeps_the_choices_and_refusals_of_before(bj):
    c, cfg, plan, blocks = _production_case(bj)
    ctx = bj.Context(0)
    try:
        for bad in (0, 3, 5, 16):
            with pytest.raises(bj.BoojumError) as e:
                ctx.set_max_row_blocks(bad)
            assert e.value.status == INVALID
        ctx.allow_recompute_plan(True)
        # a limit that row blocks would meet: refused, naming the one-block recompute plan
        ctx.set_memory_limit((blocks[1] + blocks[2]) // 2)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, 8, cfg)
        assert e.value.status == OOM and str(blocks[1]) + " bytes on the recompute plan" in str(e.value)
        assert str(blocks[2]) not in str(e.value)
        assert ctx.launch_count() == before
        ctx.set_memory_limit(blocks[1])
        nat = _setup(ctx, c, 8, cfg)
        assert nat.plan == "recompute" and nat.row_blocks == 1
        assert sum(nat.memory_plan()[k] for k in ("pool", "outside_pool")) == plan["recompute"]
        nat.close()
        # the switch set back to 1 is the default
        ctx.set_max_row_blocks(8)
        ctx.set_max_row_blocks(1)
        ctx.set_memory_limit((blocks[1] + blocks[2]) // 2)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, 8, cfg)
        assert e.value.status == OOM
        # without the recompute switch the row-block switch changes nothing either
        ctx.allow_recompute_plan(False)
        ctx.set_max_row_blocks(8)
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, 8, cfg)
        assert e.value.status == OOM and "recompute" not in str(e.value)
        assert ctx.launch_count() == before
    finally:
        ctx.close()


def test_lane_and_witness_slot_proofs_on_row_blocks(bj):
    """a lane inherits the switch and proves the parent's row-block setup; witness slots count the row-block plan; both give
    the bytes bj_prove on the parent gives"""
    cs = _production(bj, 11, witness_seeds=(701, 702))
    cfg = _cfg(2, 32)
    B4 = _blocks(bj, 11, cs[0], 8, cfg, 4)
    ctx = bj.Context(0)
    try:
        ctx.allow_recompute_plan(True)
        ctx.set_max_row_blocks(4)
        ctx.set_memory_limit(B4)
        nat = _setup(ctx, cs[0], 8, cfg)
        assert nat.plan == "recompute" and nat.row_blocks == 4
        want = [nat.prove(c["variables"], _mult(c), as_json=True) for c in cs]
        assert want[0] != want[1]
        lp = nat.memory_plan_lanes(1)
        lanes_h = bj.proof_memory_plan_lanes(11, 155, cs[0]["constants"].shape[0], 8, cfg, "recompute", 1, lookup=_lk(cs[0]), row_blocks=4)
        assert lp["total"] == lanes_h["total"] == B4 and lp["setup"] == lanes_h["setup"]
        # the parent and one lane: the setup part and two lane parts
        ctx.set_memory_limit(nat.memory_plan_lanes(2)["total"])
        lane = ctx.lane()
        lane.memory_high_water(reset=True)
        assert nat.prove(cs[1]["variables"], _mult(cs[1]), as_json=True, ctx=lane) == want[1]
        assert nat.prove(cs[0]["variables"], _mult(cs[0]), as_json=True, ctx=lane) == want[0]
        assert lane.memory_high_water() == lp["lane_pool"]
        lane.close()
        slot_bytes = bj.witness_slots_bytes(11, 155, 2, lookup=_lk(cs[0]))
        ctx.set_memory_limit(B4 + slot_bytes - 1)
        with pytest.raises(bj.BoojumError) as e:
            nat.witness_slots(2)
        assert e.value.status == OOM and str(B4) in str(e.value)
        ctx.set_memory_limit(B4 + slot_bytes)
        slots = nat.witness_slots(2)
        hw = [(bj.to_numpy(c["variables"]), bj.to_numpy(c["lookup"]["multiplicities"])) for c in cs]
        assert list(nat.prove_stream(hw + hw[::-1], slots=slots)) == want + want[::-1]
        vk = nat.vk()
        assert all(OV.verify(vk, json.loads(p)) for p in want)
        slots.close()
        nat.close()
    finally:
        ctx.close()
