"""Proving on the recompute plan on a sharded context: every rank keeps no coset of the setup, witness or stage-2 columns and
works on its own units u = rank (mod world) - whole cosets on a coset shard (world <= L), row blocks on a split shard (world
> L).  Its trees are built one committed unit at a time, its quotient units are evaluated one at a time from the natural-order
columns, and the openings, DEEP and the query answers rebuild the units they read.  The plan is opt-in per context
(Context.allow_sharded_recompute_plan); with it on, a rank limited to its recompute plan chooses it.  The ranks run as threads
on one GPU over the local transport.  Every rank's proof must be the single-GPU resident proof byte for byte, the verifier
must accept it, and every rank's pool must reach exactly its planned peak.  With the switch off the same limit is refused as
before, and a context without a communicator ignores the switch."""
import json
import threading

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


def _production(bj, log_n):
    """synthetic.generate_production_shaped: 155 columns, Q = 8, 8 lookups of width 3, 4 public inputs"""
    from era_boojum_b200 import synthetic
    ctx = bj.Context(0)
    c = synthetic.generate_production_shaped(ctx, log_n, seed=70 + log_n)
    ctx.synchronize()
    ctx.close()
    c["Q"] = c["quotient_degree"]
    return c


def _sha(bj, log_n, V, Q, pis):
    """the oracle's SHA-shaped circuit with its lookup argument on the device (Q = 4: the bench's gates)"""
    from era_boojum_b200 import synthetic
    from oracle import circuits
    c = circuits.sha_shaped(log_n, V, seed=500 + log_n, lookup=True)
    lk = dict(c["lookup"], tables=bj.to_device(c["lookup"]["tables"]), multiplicities=bj.to_device(c["lookup"]["multiplicities"]))
    return dict(variables=bj.to_device(c["variables"]), sigmas=bj.to_device(c["sigmas"]), constants=bj.to_device(c["constants"]),
                gates=synthetic.sha_shaped_gates(V), Q=Q, lookup=lk, public_inputs=list(pis))


def _shape(bj, shape, log_n):
    if shape == "production":
        return _production(bj, log_n)
    return _sha(bj, log_n, 20, 4, [(1, 3), (5, 3)] if shape == "bench" else [(2, 100)])


def _lk(c):
    return dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"]) if c["lookup"] else None


def _log_n(c):
    return c["sigmas"].shape[1].bit_length() - 1


def _plan(bj, c, cfg, world):
    return bj.proof_memory_plan(_log_n(c), c["sigmas"].shape[0], c["constants"].shape[0], c["Q"], cfg, lookup=_lk(c), world=world)


def _recompute(bj, c, cfg, world):
    return bj.proof_memory_plan_recompute_sharded(_log_n(c), c["sigmas"].shape[0], c["constants"].shape[0], c["Q"], cfg, world,
                                                  lookup=_lk(c))


def _setup(ctx, c, cfg):
    return ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["Q"], cfg, lookup=c["lookup"], public_inputs=c["public_inputs"])


def _single(bj, c, cfg):
    """the single-GPU resident proof (JSON text) and its verification key"""
    ctx = bj.Context(0)
    try:
        nat = _setup(ctx, c, cfg)
        assert nat.plan == "resident"
        proof = nat.prove(c["variables"], c["lookup"]["multiplicities"] if c["lookup"] else None, as_json=True)
        vk = nat.vk()
        nat.close()
        ctx.synchronize()
        return proof, vk
    finally:
        ctx.close()


def _sharded(bj, c, cfg, world, limits, allow):
    """bj_setup_create + bj_prove on `world` thread ranks over the local transport, rank r under limits[r] (0: the device) with
    the sharded recompute switch allow[r] -> per rank dict(plan, proof JSON, pool high-water, memory_plan())"""
    group = bj.Comm.local_group(world)
    out, errs = [None] * world, []

    def run(rank):
        try:
            ctx = bj.Context(0)
            comm = bj.Comm.local(ctx, group, rank, world, cfg.fri_lde_factor)
            ctx.set_memory_limit(limits[rank])
            ctx.allow_sharded_recompute_plan(allow[rank])
            nat = _setup(ctx, c, cfg)
            proof = nat.prove(c["variables"], c["lookup"]["multiplicities"] if c["lookup"] else None, as_json=True)
            ctx.synchronize()
            out[rank] = dict(plan=nat.plan, proof=proof, high=ctx.memory_high_water(), mp=nat.memory_plan())
            nat.close()
            comm.close()
            ctx.close()
        except BaseException as e:
            errs.append(e)

    ts = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(world)]
    [t.start() for t in ts]
    [t.join(timeout=900) for t in ts]
    if errs:
        raise errs[0]
    assert all(o is not None for o in out), "a rank did not finish"
    bj.Comm.destroy_local_group(group)
    return out


# bench: Q = 4 < L = 8 (coset shards); q_equals_l: Q = L = 4 (split from 8); production: Q = 8 > L = 2 (split from 4)
CFG = {"bench": (8, 16), "q_equals_l": (4, 16), "production": (2, 32)}


@pytest.mark.parametrize("shape,log_n,world,hasher", [
    ("production", 12, 2, "poseidon2"),
    ("production", 12, 4, "blake2s"),
    ("production", 13, 8, "keccak256"),
    ("production", 12, 16, "poseidon2"),
    ("bench", 10, 2, "keccak256"),
    ("bench", 10, 4, "poseidon2"),
    ("q_equals_l", 11, 2, "blake2s"),
    ("q_equals_l", 11, 8, "keccak256"),
    ("q_equals_l", 11, 16, "poseidon2")])
def test_sharded_recompute_plan_proves_the_single_gpu_proof(bj, shape, log_n, world, hasher):
    """at world = L with Q <= L (q_equals_l on 4 ranks) a resident rank holds one coset of every column, less than the
    recompute plan's natural-order stage-2 columns and quotient scratch: the plan saves nothing there.  With Q < L and more
    ranks than quotient units (bench on 8 and 16 ranks) some rank would own no quotient unit: the plan does not apply"""
    from era_boojum_b200 import prover
    c = _shape(bj, shape, log_n)
    L, cap = CFG[shape]
    cfg = prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100, hasher=hasher, transcript=hasher)
    plan = _plan(bj, c, cfg, world)
    limit = _recompute(bj, c, cfg, world)
    assert limit < min(p for p in (plan["resident"], plan["streamed_sharded"]) if p)

    want, vk = _single(bj, c, cfg)
    assert OV.verify(vk, json.loads(want))
    for rank, r in enumerate(_sharded(bj, c, cfg, world, [limit] * world, [True] * world)):
        assert r["plan"] == "recompute", rank
        # the chunk grows as far as the pool peak does not move
        assert r["mp"]["pool"] + r["mp"]["outside_pool"] == limit and 2 <= r["mp"]["chunk"] <= 16
        assert r["high"] == r["mp"]["pool"], (rank, r["high"], r["mp"])
        assert r["proof"] == want, rank


def test_ranks_under_different_limits_agree_on_the_recompute_plan(bj):
    """production shape on 4 ranks (2 row blocks per coset) with the switch on every rank: rank 0 could take the resident plan,
    rank 1 the streamed one, ranks 2 and 3 only the recompute plan.  The resident and streamed plans exchange their LDEs'
    monomials and the recompute plan does not, so the ranks agree before their first collective: every rank takes the
    recompute plan (the group runs at its slowest rank's pace anyway) and returns the single-GPU proof"""
    from era_boojum_b200 import prover
    c = _production(bj, 12)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    plan = _plan(bj, c, cfg, 4)
    rec = _recompute(bj, c, cfg, 4)
    want, _ = _single(bj, c, cfg)
    limits = [0, (plan["streamed_sharded"] + plan["resident"]) // 2, rec, rec]
    res = _sharded(bj, c, cfg, 4, limits, [True] * 4)
    assert [r["plan"] for r in res] == ["recompute"] * 4
    for rank, r in enumerate(res):
        assert r["high"] == r["mp"]["pool"], (rank, r["high"], r["mp"])
        assert r["proof"] == want, rank


def test_ranks_keep_their_plans_while_none_needs_the_recompute_plan(bj):
    """the switch on every rank, rank 0 resident, rank 1 streamed: the agreement changes nothing"""
    from era_boojum_b200 import prover
    c = _production(bj, 12)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    plan = _plan(bj, c, cfg, 2)
    want, _ = _single(bj, c, cfg)
    res = _sharded(bj, c, cfg, 2, [0, (plan["streamed_sharded"] + plan["resident"]) // 2], [True, True])
    assert [r["plan"] for r in res] == ["resident", "streamed"]
    assert all(r["proof"] == want for r in res)


def _refused_setup(bj, c, cfg, world, limit, allow):
    """rank 0 of a `world`-rank context alone: bj_setup_create must refuse before its first collective -> (error, launches)"""
    group = bj.Comm.local_group(world)
    ctx = bj.Context(0)
    comm = bj.Comm.local(ctx, group, 0, world, cfg.fri_lde_factor)
    result = []

    def setup():
        try:
            result.append(_setup(ctx, c, cfg))
        except bj.BoojumError as e:
            result.append(e)

    try:
        ctx.set_memory_limit(limit)
        ctx.allow_sharded_recompute_plan(allow)
        before = ctx.launch_count()
        t = threading.Thread(target=setup, daemon=True)
        t.start()
        t.join(timeout=120)
        assert not t.is_alive(), "bj_setup_create did not refuse before its first collective"
        return result[0], ctx.launch_count() - before
    finally:
        comm.close()
        ctx.close()
        bj.Comm.destroy_local_group(group)


@pytest.mark.parametrize("shape,world", [("production", 2), ("production", 4), ("q_equals_l", 8)])
def test_the_switch_off_keeps_the_refusal(bj, shape, world):
    """the recompute plan's limit without the switch: BJ_ERR_OOM before any launch, the message of before (no recompute bytes)"""
    from era_boojum_b200 import prover
    c = _shape(bj, shape, 10)
    L, cap = CFG[shape]
    cfg = prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100)
    plan, rec = _plan(bj, c, cfg, world), _recompute(bj, c, cfg, world)
    e, launches = _refused_setup(bj, c, cfg, world, rec, False)
    assert isinstance(e, bj.BoojumError) and e.status == OOM
    msg = str(e)
    assert str(plan["resident"]) in msg and "recompute" not in msg   # the limit itself is the recompute plan's bytes
    if plan["streamed_sharded"]:
        assert str(plan["streamed_sharded"]) in msg
    assert launches == 0


@pytest.mark.parametrize("world", [2, 16])
def test_limit_below_the_sharded_recompute_plan_is_refused(bj, world):
    """one byte below the plan with the switch on: BJ_ERR_OOM naming the recompute bytes, nothing launched"""
    from era_boojum_b200 import prover
    c = _production(bj, 10)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    plan, rec = _plan(bj, c, cfg, world), _recompute(bj, c, cfg, world)
    e, launches = _refused_setup(bj, c, cfg, world, rec - 1, True)
    assert isinstance(e, bj.BoojumError) and e.status == OOM
    msg = str(e)
    assert str(plan["resident"]) in msg and str(plan["streamed_sharded"]) in msg and str(rec) in msg and "recompute" in msg
    assert launches == 0


def test_a_context_without_a_communicator_ignores_the_switch(bj):
    """one GPU, Q = L: under the one-GPU recompute plan's limit only bj_ctx_allow_recompute_plan makes the plan available"""
    from era_boojum_b200 import prover
    c = _shape(bj, "q_equals_l", 10)
    cfg = prover.ProofConfig(fri_lde_factor=4, merkle_tree_cap_size=16, security_level=100)
    plan = _plan(bj, c, cfg, 1)
    assert plan["compact"] is None and plan["streamed"] is None
    ctx = bj.Context(0)
    try:
        ctx.set_memory_limit((plan["recompute"] + plan["resident"]) // 2)
        ctx.allow_sharded_recompute_plan(True)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            _setup(ctx, c, cfg)
        assert e.value.status == OOM
        assert "recompute" not in str(e.value) and str(plan["recompute"]) not in str(e.value)
        assert ctx.launch_count() == before
        ctx.allow_recompute_plan(True)
        nat = _setup(ctx, c, cfg)
        assert nat.plan == "recompute"
        nat.close()
    finally:
        ctx.close()
