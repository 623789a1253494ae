"""Proof lanes: several proofs of one setup in flight on one GPU.  A lane (Context.lane, bj_ctx_create_lane) is a context on the
parent's device with its own stream and pool that proves against the parent's setups.  Distinct witnesses of one setup are
proved on 2, 3 and 4 lanes driven from host threads at the same time, on the bench- and production-shaped circuits, on each
memory plan (forced with a device-memory limit and the recompute switch) and with every tree hasher / transcript pair.  Every
lane proof must be byte for byte the proof bj_prove gives on the parent, which the verifier accepts; a fresh lane's pool must
peak at the lane part of bj_proof_memory_plan_lanes and stay there through a second round of proofs; and the refusals (sharded parent, memory limit, teardown order) must hold with nothing launched."""
import ctypes
import json
import threading

import pytest

from oracle import verifier as OV

pytestmark = pytest.mark.gpu

INVALID, OOM = -1, -4  # BJ_ERR_INVALID_ARG, BJ_ERR_OOM
K = 4                  # witnesses per setup


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


_WITNESSES = {}


def _witnesses(bj, shape, log_n):
    """K circuits of one structure (same sigmas, constants and tables) with pairwise different witnesses (device tensors)"""
    key = (shape, log_n)
    if key not in _WITNESSES:
        from era_boojum_b200 import synthetic
        ctx = bj.Context(0)
        out = []
        for ws in range(K):
            if shape == "production":
                out.append(synthetic.generate_production_shaped(ctx, log_n, seed=90 + log_n, witness_seed=700 + ws))
            else:
                v, s, c, g, q, lk = synthetic.generate(ctx, log_n, 60, seed=30 + log_n, lookup=True, witness_seed=800 + ws)
                out.append(dict(variables=v, sigmas=s, constants=c, gates=g, quotient_degree=q, lookup=lk, public_inputs=[(3, 5)]))
        ctx.synchronize()
        ctx.close()
        _WITNESSES[key] = out
    return _WITNESSES[key]


def _cfg(shape, hasher="poseidon2", transcript="poseidon2"):
    from era_boojum_b200 import prover
    L, cap = (2, 32) if shape == "production" else (8, 16)
    return prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100, hasher=hasher, transcript=transcript)


def _plan_limit(bj, shape, log_n, c, cfg, plan):
    """the device-memory limit under which bj_setup_create chooses `plan` (0: the resident plan under the device's memory)"""
    lk = c["lookup"]
    lk = dict(width=lk["width"], num_repetitions=lk["num_repetitions"])
    p = bj.proof_memory_plan(log_n, c["sigmas"].shape[0], c["constants"].shape[0], c["quotient_degree"], cfg, lookup=lk)
    if plan == "resident":
        return 0
    if plan == "recompute":
        return (p["recompute"] + min(p[k] for k in ("resident", "compact", "streamed") if p[k])) // 2
    return (p[plan] + p["resident"]) // 2


def _setup(ctx, c, cfg):
    return ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                            public_inputs=c["public_inputs"])


def _parent(bj, shape, log_n, cfg, plan):
    """a context whose setup is on `plan`; the limit is then lifted so that lanes fit beside it (the setup keeps its plan)"""
    cs = _witnesses(bj, shape, log_n)
    ctx = bj.Context(0)
    ctx.set_memory_limit(_plan_limit(bj, shape, log_n, cs[0], cfg, plan))
    ctx.allow_recompute_plan(plan == "recompute")
    nat = _setup(ctx, cs[0], cfg)
    assert nat.plan == plan
    import torch
    ctx.set_memory_limit(torch.cuda.get_device_properties(0).total_memory)
    return ctx, nat, cs


def _on_lanes(nat, lanes, cs):
    """proves witness i on lane i % len(lanes), every lane from its own thread, all started together -> proofs in order"""
    out = [None] * len(cs)
    errors = []
    start = threading.Barrier(len(lanes))

    def run(k):
        try:
            start.wait()
            for i in range(k, len(cs), len(lanes)):
                out[i] = nat.prove(cs[i]["variables"], cs[i]["lookup"]["multiplicities"], as_json=True, ctx=lanes[k])
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(k,)) for k in range(len(lanes))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    return out


@pytest.mark.parametrize("shape,log_n,plan", [
    ("bench", 12, "resident"), ("bench", 12, "compact"), ("bench", 12, "recompute"),
    ("production", 10, "resident"), ("production", 10, "streamed"), ("production", 10, "recompute")])
def test_lanes_prove_the_parent_proofs_on_every_plan(bj, shape, log_n, plan):
    cfg = _cfg(shape)
    ctx, nat, cs = _parent(bj, shape, log_n, cfg, plan)
    try:
        want = [nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in cs]
        assert len(set(want)) == K
        assert OV.verify(nat.vk(), json.loads(want[0]))
        for n_lanes in (2, 3, 4):
            lanes = [ctx.lane() for _ in range(n_lanes)]
            got = _on_lanes(nat, lanes, cs)
            assert got == want, (n_lanes, [g == w for g, w in zip(got, want)])
            mp = nat.memory_plan_lanes(n_lanes)
            for ln in lanes:
                # a fresh lane's pool peaks at the lane part of the plan
                assert ln.memory_high_water() == mp["lane_pool"], (ln.memory_high_water(), mp)
            # a second round on the same lanes: the same proofs, and no lane's pool grows past its first peak
            assert _on_lanes(nat, lanes, cs) == want
            for ln in lanes:
                assert ln.memory_high_water() == mp["lane_pool"]
            for ln in lanes:
                ln.close()
        assert mp["setup"] + mp["lane"] == sum(nat.memory_plan()[k] for k in ("pool", "outside_pool"))
    finally:
        nat.close()
        ctx.close()


@pytest.mark.parametrize("shape,log_n,plan", [
    ("bench", 12, "resident"), ("bench", 12, "compact"), ("bench", 12, "recompute"),
    ("production", 10, "resident"), ("production", 10, "streamed"), ("production", 10, "recompute")])
def test_lanes_from_a_cold_cache(bj, shape, log_n, plan):
    """lanes created right after bj_setup_create, before any proof on the parent: the lanes build the coset-power tables the
    setup did not need into the parent's cache (several missing the same table at once), and a lane whose transforms are
    longer than the parent's twiddle pair (streamed and recompute plans: the quotient's n * Q) builds a private pair.  The
    parent's proofs are taken afterwards."""
    cfg = _cfg(shape)
    ctx, nat, cs = _parent(bj, shape, log_n, cfg, plan)
    try:
        lanes = [ctx.lane() for _ in range(4)]
        got = _on_lanes(nat, lanes, cs)
        for ln in lanes:
            ln.close()
        want = [nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in cs]
        assert got == want, [g == w for g, w in zip(got, want)]
        assert OV.verify(nat.vk(), json.loads(got[2]))
    finally:
        nat.close()
        ctx.close()


def test_parent_grows_its_tables_while_lanes_prove(bj):
    """the parent creates and proves a larger setup while its lanes prove a smaller one: the parent's twiddle pair grows and the
    replaced pair is retired, not freed, under the lanes; once the lanes are gone the parent's next proof frees it"""
    cfg = _cfg("bench")
    small = _witnesses(bj, "bench", 10)
    big = _witnesses(bj, "bench", 13)
    ctx = bj.Context(0)
    try:
        nat = _setup(ctx, small[0], cfg)
        lanes = [ctx.lane() for _ in range(3)]
        nat_big = _setup(ctx, big[0], cfg)  # grows the parent's twiddles with the lanes alive
        got, got_big, errors = [None] * K, [None] * K, []

        def parent():
            try:
                for i in range(K):
                    got_big[i] = nat_big.prove(big[i]["variables"], big[i]["lookup"]["multiplicities"], as_json=True)
            except Exception as e:  # noqa: BLE001 - reported below
                errors.append(e)

        t = threading.Thread(target=parent)
        t.start()
        got = _on_lanes(nat, lanes, small)
        t.join()
        assert not errors, errors
        for ln in lanes:
            ln.close()
        want_big = [nat_big.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in big]
        want = [nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in small]
        assert got == want
        assert got_big == want_big
        assert OV.verify(nat_big.vk(), json.loads(got_big[0]))
        nat_big.close()
        nat.close()
    finally:
        ctx.close()


@pytest.mark.parametrize("hasher,transcript", [("poseidon2", "poseidon2"), ("blake2s", "blake2s"), ("keccak256", "keccak256"),
                                               ("poseidon2", "poseidon")])
@pytest.mark.parametrize("shape,log_n", [("bench", 11), ("production", 9)])
def test_lanes_with_every_hasher_and_transcript(bj, shape, log_n, hasher, transcript):
    cfg = _cfg(shape, hasher, transcript)
    ctx, nat, cs = _parent(bj, shape, log_n, cfg, "resident")
    try:
        want = [nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in cs]
        lanes = [ctx.lane() for _ in range(3)]
        assert _on_lanes(nat, lanes, cs) == want
        assert OV.verify(nat.vk(), json.loads(want[1]))
        for ln in lanes:
            ln.close()
    finally:
        nat.close()
        ctx.close()


def test_prove_concurrent_yields_the_proofs_in_order(bj):
    cfg = _cfg("bench")
    ctx, nat, cs = _parent(bj, "bench", 11, cfg, "resident")
    try:
        want = [nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in cs]
        ws = [(c["variables"], c["lookup"]["multiplicities"]) for c in cs]
        assert list(nat.prove_concurrent(ws + ws, lanes=3)) == want + want
        assert list(nat.prove_concurrent(iter(ws[:2]), lanes=2, as_json=False)) == [json.loads(w) for w in want[:2]]
        # prove_concurrent closed its lanes: the parent is no longer refused
        nat.close()
        assert bj.native.lib.bj_ctx_destroy(ctx._h) == 0
        ctx._h = None
    finally:
        nat.close()
        ctx.close()


def test_lane_refusals(bj):
    lib = bj.native.lib
    cfg = _cfg("bench")
    cs = _witnesses(bj, "bench", 11)
    # a sharded parent has no lanes
    ctx = bj.Context(0)
    ctx.set_domain_shard(0, 2, 8)
    h = ctypes.c_void_p()
    assert lib.bj_ctx_create_lane(ctx._h, ctypes.byref(h)) == INVALID and not h.value
    assert b"sharded" in lib.bj_last_error(ctx._h)
    ctx.close()

    ctx = bj.Context(0)
    nat = _setup(ctx, cs[0], cfg)
    try:
        # over the limit: the parent and one lane need plan_lanes(2)["total"]; one byte less is refused before any launch
        total = nat.memory_plan_lanes(2)["total"]
        ctx.set_memory_limit(total - 1)
        launches = ctx.launch_count()
        assert lib.bj_ctx_create_lane(ctx._h, ctypes.byref(h)) == OOM and not h.value
        msg = lib.bj_last_error(ctx._h).decode()
        assert str(total) in msg and str(total - 1) in msg, msg
        assert ctx.launch_count() == launches
        ctx.set_memory_limit(total)
        lane = ctx.lane()
        assert lib.bj_ctx_create_lane(ctx._h, ctypes.byref(h)) == OOM  # a second lane does not fit
        ctx.set_memory_limit(0)
        # a lane inherits the limit it was created under, creates no setup and has no lanes
        with pytest.raises(bj.BoojumError, match="create the setup on the parent"):
            _setup(lane, cs[0], cfg)
        assert lib.bj_ctx_create_lane(lane._h, ctypes.byref(h)) == INVALID
        assert lib.bj_ctx_set_stream(lane._h, None) == INVALID
        # a lane proves only against its parent's setups
        other = bj.Context(0)
        assert lib.bj_prove(other._h, nat._h, lane._ptr(cs[0]["variables"]), lane._ptr(cs[0]["lookup"]["multiplicities"]),
                            ctypes.byref(h)) == INVALID
        other.close()

        # teardown: the parent is refused while a lane is alive, and stays usable
        assert lib.bj_ctx_destroy(ctx._h) == INVALID
        assert b"lane" in lib.bj_last_error(ctx._h)
        want = nat.prove(cs[1]["variables"], cs[1]["lookup"]["multiplicities"], as_json=True)
        assert nat.prove(cs[1]["variables"], cs[1]["lookup"]["multiplicities"], as_json=True, ctx=lane) == want
        # a setup created with a lane alive counts the lane: under a limit of the resident plan alone it takes the compact plan
        # if that and a lane fit, else it is refused
        lk = dict(width=cs[0]["lookup"]["width"], num_repetitions=cs[0]["lookup"]["num_repetitions"])
        shape = (11, cs[0]["sigmas"].shape[0], cs[0]["constants"].shape[0], cs[0]["quotient_degree"], cfg)
        resident = bj.proof_memory_plan(*shape, lookup=lk)["resident"]
        compact = bj.proof_memory_plan_lanes(*shape, "compact", 2, lookup=lk)
        ctx.set_memory_limit(resident)
        if compact["total"] <= resident:
            extra = _setup(ctx, cs[0], cfg)
            assert extra.plan == "compact"
            extra.close()
        else:
            with pytest.raises(bj.BoojumError, match="lane"):
                _setup(ctx, cs[0], cfg)
        ctx.set_memory_limit(0)
        # a setup is freed once the proofs that read it have returned; the lane goes on with a new setup of its parent
        nat.close()
        nat = _setup(ctx, cs[0], cfg)
        assert nat.prove(cs[1]["variables"], cs[1]["lookup"]["multiplicities"], as_json=True, ctx=lane) == want
        lane.close()
        assert lib.bj_ctx_destroy(None) == 0
    finally:
        nat.close()
        ctx.close()
    assert ctx._h is None
