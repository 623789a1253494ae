"""Proving under a device-memory limit on a sharded context when the quotient degree Q exceeds the LDE factor L.  A per-rank
limit between the sharded streamed plan and the sharded resident plan makes every rank's bj_setup_create choose the streamed
plan: each rank evaluates its units of the committed cosets [0, L) only, and its quotient units of cosets [L, Q) one at a time
(whole cosets on a coset shard, world <= L; row blocks on a split shard, world > L).  The ranks run as threads on one GPU over
the local transport.  Every rank's proof must be the single-GPU resident proof byte for byte, the verifier must accept it,
and every rank's pool must stay within its planned peak."""
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
    return c


def _bench(bj, log_n, V, lookup, pis):
    """synthetic.generate: the SHA-bench-shaped circuit, Q = 4"""
    from era_boojum_b200 import synthetic
    ctx = bj.Context(0)
    gen = synthetic.generate(ctx, log_n, V, seed=11 + log_n, lookup=lookup)
    ctx.synchronize()
    ctx.close()
    return dict(variables=gen[0], sigmas=gen[1], constants=gen[2], gates=gen[3], quotient_degree=gen[4],
                lookup=gen[5] if lookup else None, public_inputs=list(pis))


def _plan(bj, c, cfg, world):
    lk = c["lookup"]
    lk = dict(width=lk["width"], num_repetitions=lk["num_repetitions"]) if lk else None
    log_n = c["sigmas"].shape[1].bit_length() - 1
    return bj.proof_memory_plan(log_n, c["sigmas"].shape[0], c["constants"].shape[0], c["quotient_degree"], cfg, lookup=lk, world=world)


def _single(bj, c, cfg):
    """the single-GPU resident proof (JSON text) and its verification key"""
    ctx = bj.Context(0)
    try:
        nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                               public_inputs=c["public_inputs"])
        assert nat.plan == "resident"
        proof = nat.prove(c["variables"], c["lookup"]["multiplicities"] if c["lookup"] else None, as_json=True)
        vk = nat.vk()
        nat.close()
        ctx.synchronize()
        return proof, vk
    finally:
        ctx.close()


def _sharded(bj, c, cfg, world, limits):
    """bj_setup_create + bj_prove on `world` thread ranks over the local transport, rank r under limits[r] (0: the device)
    -> per rank dict(plan, proof JSON, pool high-water, memory_plan())"""
    group = bj.Comm.local_group(world)
    out, errs = [None] * world, []

    def run(rank):
        try:
            ctx = bj.Context(0)
            comm = bj.Comm.local(ctx, group, rank, world, cfg.fri_lde_factor)
            ctx.set_memory_limit(limits[rank])
            nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                                   public_inputs=c["public_inputs"])
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


@pytest.mark.parametrize("shape,log_n,world,hasher", [
    ("production", 12, 2, "poseidon2"),
    ("production", 12, 4, "blake2s"),
    ("production", 13, 8, "poseidon2"),
    ("production", 12, 16, "blake2s"),
    ("bench", 10, 2, "blake2s"),
    ("bench", 11, 4, "poseidon2"),
    ("bench", 10, 8, "blake2s"),
    ("bench", 10, 16, "poseidon2")])
def test_sharded_streamed_plan_proves_the_single_gpu_proof(bj, shape, log_n, world, hasher):
    """L = 2: world 2 is a coset shard, 4, 8 and 16 split every coset into 2, 4 and 8 row blocks"""
    from era_boojum_b200 import prover
    c = _production(bj, log_n) if shape == "production" else _bench(bj, log_n, 60, log_n != 11, [(1, 3), (5, 3)] if log_n == 11 else [])
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32 if shape == "production" else 16, security_level=100,
                             hasher=hasher, transcript=hasher)
    assert c["quotient_degree"] > cfg.fri_lde_factor
    plan = _plan(bj, c, cfg, world)
    assert plan["streamed"] is None and plan["streamed_sharded"] is not None and plan["streamed_sharded"] < plan["resident"]
    limit = (plan["streamed_sharded"] + plan["resident"]) // 2

    want, vk = _single(bj, c, cfg)
    assert OV.verify(vk, json.loads(want))
    for rank, r in enumerate(_sharded(bj, c, cfg, world, [limit] * world)):
        assert r["plan"] == "streamed", rank
        assert r["mp"]["pool"] + r["mp"]["outside_pool"] == plan["streamed_sharded"] <= limit and r["mp"]["chunk"] == 0
        assert r["high"] <= r["mp"]["pool"], (rank, r["high"], r["mp"])
        assert r["proof"] == want, rank


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_on_different_plans_agree(bj, world):
    """rank 0 under a limit (streamed), the others on the resident plan: the plans keep the same committed units and run the
    same collectives, so every rank still returns the single-GPU proof"""
    from era_boojum_b200 import prover
    c = _bench(bj, 10, 60, True, [(2, 7)])
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=16, security_level=100)
    plan = _plan(bj, c, cfg, world)
    want, _ = _single(bj, c, cfg)
    res = _sharded(bj, c, cfg, world, [(plan["streamed_sharded"] + plan["resident"]) // 2] + [0] * (world - 1))
    assert [r["plan"] for r in res] == ["streamed"] + ["resident"] * (world - 1)
    for rank, r in enumerate(res):
        assert r["high"] <= r["mp"]["pool"], (rank, r["high"], r["mp"])
        assert r["proof"] == want, rank


def test_limit_below_the_sharded_streamed_plan_is_refused(bj):
    """one byte below the plan on rank 0 of a 4-rank context: refused with BJ_ERR_OOM before the first collective (the
    other ranks never join) and before any kernel"""
    from era_boojum_b200 import prover
    c = _production(bj, 10)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    plan = _plan(bj, c, cfg, 4)
    group = bj.Comm.local_group(4)
    ctx = bj.Context(0)
    comm = bj.Comm.local(ctx, group, 0, 4, 2)
    result = []

    def setup():
        try:
            result.append(ctx.native_setup(c["sigmas"], c["constants"], c["gates"], 8, cfg, lookup=c["lookup"],
                                           public_inputs=c["public_inputs"]))
        except bj.BoojumError as e:
            result.append(e)

    try:
        ctx.set_memory_limit(plan["streamed_sharded"] - 1)
        before = ctx.launch_count()
        t = threading.Thread(target=setup, daemon=True)
        t.start()
        t.join(timeout=120)
        assert not t.is_alive(), "bj_setup_create did not refuse before its first collective"
        e = result[0]
        assert isinstance(e, bj.BoojumError) and e.status == OOM
        assert str(plan["resident"]) in str(e) and str(plan["streamed_sharded"]) in str(e)
        assert ctx.launch_count() == before
    finally:
        comm.close()
        ctx.close()
        bj.Comm.destroy_local_group(group)
