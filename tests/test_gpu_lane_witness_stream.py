"""Witness slot sets on proof lanes: each lane (Context.lane) streams host witnesses through its own slot set
(NativeSetup.witness_slots(..., ctx=lane)) on its own copy stream while it proves, all lanes from their own threads at once.
Several pairwise different witnesses of one setup are streamed on 2 and 3 lanes with 1 and 2 slots each (more witnesses than
slots), from pinned and pageable host memory, as columns and as the reference's WitnessVec, on the resident, compact, streamed,
recompute and row-block recompute plans.  Every proof must be byte for byte the proof bj_prove gives on the parent, which the
verifier accepts; each lane's pool must peak at its proof part plus its set; the memory checks must count every set exactly;
and the refusals (a set of another context, a setup of another parent, a hint replaced or a lane destroyed under a live set)
must hold with nothing launched."""
import ctypes
import json
import threading

import numpy as np
import pytest

from oracle import verifier as OV

pytestmark = pytest.mark.gpu

INVALID, OOM = -1, -4  # BJ_ERR_INVALID_ARG, BJ_ERR_OOM
K = 5                  # witnesses per setup


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
        import torch
        from era_boojum_b200 import synthetic
        ctx = bj.Context(0)
        out = []
        for ws in range(K):
            if shape == "production":
                out.append(synthetic.generate_production_shaped(ctx, log_n, seed=90 + log_n, witness_seed=900 + ws))
            else:
                v, s, c, g, q, lk = synthetic.generate(ctx, log_n, 60, seed=30 + log_n, lookup=True, witness_seed=950 + ws)
                out.append(dict(variables=v, sigmas=s, constants=c, gates=g, quotient_degree=q, lookup=lk, public_inputs=[(3, 5)]))
        ctx.synchronize()
        ctx.close()
        for c in out[1:]:
            assert torch.equal(c["sigmas"], out[0]["sigmas"]) and torch.equal(c["lookup"]["tables"], out[0]["lookup"]["tables"])
        _WITNESSES[key] = out
    return _WITNESSES[key]


def _cfg(shape):
    from era_boojum_b200 import prover
    L, cap = (2, 32) if shape == "production" else (8, 16)
    return prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=cap, security_level=100)


def _lk(c):
    return dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"])


def _setup(ctx, c, cfg):
    return ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                            public_inputs=c["public_inputs"])


def _parent(bj, shape, log_n, plan):
    """a context whose setup is on `plan` ("recompute_blocks": the recompute plan in 2 row blocks); the limit is then lifted
    so that lanes and their sets fit beside it (the setup keeps its plan)"""
    import torch
    cs = _witnesses(bj, shape, log_n)
    c, cfg = cs[0], _cfg(shape)
    shp = (log_n, c["sigmas"].shape[0], c["constants"].shape[0], c["quotient_degree"], cfg)
    p = bj.proof_memory_plan(*shp, lookup=_lk(c))
    ctx = bj.Context(0)
    if plan == "recompute_blocks":
        ctx.allow_recompute_plan(True)
        ctx.set_max_row_blocks(2)
        ctx.set_memory_limit((bj.proof_memory_plan_recompute_blocks(*shp, 2, lookup=_lk(c)) + p["recompute"]) // 2)
    elif plan == "recompute":
        ctx.allow_recompute_plan(True)
        ctx.set_memory_limit((p["recompute"] + min(p[k] for k in ("resident", "compact", "streamed") if p[k])) // 2)
    elif plan != "resident":
        ctx.set_memory_limit((p[plan] + p["resident"]) // 2)
    nat = _setup(ctx, c, cfg)
    assert nat.plan == ("recompute" if plan == "recompute_blocks" else plan)
    assert nat.row_blocks == (2 if plan == "recompute_blocks" else 1)
    ctx.set_memory_limit(torch.cuda.get_device_properties(0).total_memory)
    return ctx, nat, cs


def _pinned(a):
    import torch
    signed = {8: (np.int64, torch.int64), 4: (np.int32, torch.int32)}[a.dtype.itemsize]
    t = torch.empty(a.shape, dtype=signed[1], pin_memory=True)
    t.copy_(torch.from_numpy(np.ascontiguousarray(a).view(signed[0])))
    assert t.is_pinned()
    return t


def _vec_hint(V, n, extra=5, seed=11):
    """a DenseVariablesCopyHint of one setup: cell (c, row) reads all_values[perm[c * n + row]]"""
    perm = np.random.default_rng(seed).permutation(V * n + extra)[: V * n]
    return perm.reshape(V, n).astype(np.uint64), V * n + extra


def _inputs(bj, cs, memory, mode, hint=None, n_values=0):
    """host witnesses: (variables, multiplicities) columns or (all_values, u32 multiplicities) WitnessVecs, pinned or pageable"""
    out = []
    for c in cs:
        v, m = bj.to_numpy(c["variables"]), bj.to_numpy(c["lookup"]["multiplicities"])
        if mode == "vec":
            av = np.full(n_values, 4321, np.uint64)
            av[hint.reshape(-1)] = v.reshape(-1)
            v, m = av, m.astype(np.uint32)
        out.append((_pinned(v), _pinned(m)) if memory == "pinned" else (v, m))
    return out


def _on_threads(jobs):
    """runs each callable on its own thread, all started together -> the results in order"""
    out, errors = [None] * len(jobs), []
    start = threading.Barrier(len(jobs))

    def run(k):
        try:
            start.wait()
            out[k] = jobs[k]()
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(k,)) for k in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    return out


def _stream_on_lanes(nat, sets, inputs):
    """witness i streamed through set i % len(sets), each set's lane on its own thread -> the proofs in input order"""
    L = len(sets)
    per = _on_threads([lambda k=k: list(nat.prove_stream([inputs[i] for i in range(k, len(inputs), L)], slots=sets[k]))
                       for k in range(L)])
    got = [None] * len(inputs)
    for k in range(L):
        for i, p in zip(range(k, len(inputs), L), per[k]):
            got[i] = p
    return got


def _want(nat, cs):
    return [nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True) for c in cs]


@pytest.mark.parametrize("shape,log_n,plan,n_lanes,n_slots,memory,mode", [
    ("production", 10, "resident", 2, 2, "pinned", "columns"),
    ("production", 10, "resident", 3, 1, "pageable", "vec"),
    ("production", 10, "streamed", 3, 2, "pageable", "columns"),
    ("production", 10, "streamed", 2, 1, "pinned", "vec"),
    ("production", 10, "recompute", 2, 2, "pinned", "vec"),
    ("production", 10, "recompute", 3, 1, "pageable", "columns"),
    ("bench", 11, "resident", 3, 2, "pinned", "vec"),
    ("bench", 11, "compact", 2, 2, "pageable", "columns"),
    ("bench", 11, "recompute_blocks", 2, 2, "pageable", "vec")])
def test_lane_streams_prove_the_parent_proofs(bj, shape, log_n, plan, n_lanes, n_slots, memory, mode):
    ctx, nat, cs = _parent(bj, shape, log_n, plan)
    try:
        want = _want(nat, cs)
        assert len(set(want)) == K
        assert OV.verify(nat.vk(), json.loads(want[0]))
        V, n = cs[0]["variables"].shape
        hint, n_values = _vec_hint(V, n)
        max_values = n_values if mode == "vec" else 0
        if mode == "vec":
            nat.attach_variables_hint(hint)
        inputs = _inputs(bj, cs, memory, mode, hint, n_values)
        lanes = [ctx.lane() for _ in range(n_lanes)]
        sets = [nat.witness_slots(n_slots, max_values, ctx=ln) for ln in lanes]
        got = _stream_on_lanes(nat, sets, inputs)
        assert got == want, [g == w for g, w in zip(got, want)]
        # each lane's pool: its set, then its proofs' peak on top
        own, _ = bj.witness_slots_bytes_split(log_n, V, n_slots, max_values, lookup=_lk(cs[0]))
        lane_pool = nat.memory_plan_lanes(1)["lane_pool"]
        for ln in lanes:
            assert ln.memory_high_water() == lane_pool + own, (ln.memory_high_water(), lane_pool, own)
        # a second round through the same sets, in another order
        order = [4, 2, 0, 3, 1]
        assert _stream_on_lanes(nat, sets, [inputs[i] for i in order]) == [want[i] for i in order]
        for ln in lanes:
            assert ln.memory_high_water() == lane_pool + own
        for s in sets:
            s.close()
        for ln in lanes:
            ln.close()
    finally:
        nat.close()
        ctx.close()


def test_parent_and_lanes_stream_at_once(bj):
    """the parent streams through its own set while two lanes stream through theirs: all proofs stay the parent's"""
    ctx, nat, cs = _parent(bj, "bench", 11, "resident")
    try:
        want = _want(nat, cs)
        V, n = cs[0]["variables"].shape
        hint, n_values = _vec_hint(V, n)
        nat.attach_variables_hint(hint)
        vec = _inputs(bj, cs, "pinned", "vec", hint, n_values)
        lanes = [ctx.lane() for _ in range(2)]
        sets = [nat.witness_slots(2, n_values, ctx=ln) for ln in lanes]
        mine = nat.witness_slots(2, n_values)
        order = [3, 1, 4, 0, 2, 1]
        jobs = [lambda: list(nat.prove_stream([vec[i] for i in order], slots=mine))]
        jobs += [lambda s=s: list(nat.prove_stream(vec, slots=s)) for s in sets]
        got = _on_threads(jobs)
        assert got[0] == [want[i] for i in order]
        assert got[1] == want and got[2] == want
        for s in sets + [mine]:
            s.close()
        for ln in lanes:
            ln.close()
    finally:
        nat.close()
        ctx.close()


def test_prove_concurrent_with_host_witnesses(bj):
    ctx, nat, cs = _parent(bj, "bench", 11, "resident")
    try:
        want = _want(nat, cs)
        assert OV.verify(nat.vk(), json.loads(want[1]))
        pinned = _inputs(bj, cs, "pinned", "columns")
        assert list(nat.prove_concurrent(pinned + pinned[:2], lanes=2, slots_per_lane=2)) == want + want[:2]
        pageable = _inputs(bj, cs, "pageable", "columns")
        assert list(nat.prove_concurrent(iter(pageable[::-1]), lanes=3, slots_per_lane=1, as_json=False)) == \
            [json.loads(w) for w in want[::-1]]
        # a mix of device and host witnesses: ValueError before any proof, no lane left behind
        device = [(c["variables"], c["lookup"]["multiplicities"]) for c in cs]
        before = ctx.launch_count()
        with pytest.raises(ValueError):
            list(nat.prove_concurrent([device[0], pinned[1]], lanes=2))
        with pytest.raises(ValueError):
            list(nat.prove_concurrent([pinned[0], device[1], pinned[2]], lanes=2))
        assert ctx.launch_count() == before
        # WitnessVecs once a hint is attached
        V, n = cs[0]["variables"].shape
        hint, n_values = _vec_hint(V, n)
        nat.attach_variables_hint(hint)
        vec = _inputs(bj, cs, "pageable", "vec", hint, n_values)
        assert list(nat.prove_concurrent(vec, lanes=2, slots_per_lane=2)) == want
        # every lane and set was closed: the parent can be destroyed
        nat.close()
        assert bj.native.lib.bj_ctx_destroy(ctx._h) == 0
        ctx._h = None
    finally:
        nat.close()
        ctx.close()


def test_lane_set_memory_is_counted_exactly(bj):
    """a set on a lane is checked against the setup with the lanes and the parent proving, the hint once, the parent's sets,
    the lanes' sets and its own bytes: at that total it is created, one byte below it is refused naming every term, with the
    lane's pool untouched and nothing launched.  A new lane then counts the lanes' sets too."""
    lib = bj.native.lib
    cs = _witnesses(bj, "bench", 11)
    c = cs[0]
    V, n = c["variables"].shape
    ctx = bj.Context(0)
    try:
        nat = _setup(ctx, c, _cfg("bench"))
        hint, n_values = _vec_hint(V, n)
        nat.attach_variables_hint(hint)
        parent_set = nat.witness_slots(1, 0)
        parent_bytes = bj.witness_slots_bytes(11, V, 1, 0, lookup=_lk(c))
        a, b = ctx.lane(), ctx.lane()
        set_a = nat.witness_slots(2, n_values, ctx=a)
        own_a, hint_bytes = bj.witness_slots_bytes_split(11, V, 2, n_values, lookup=_lk(c))
        assert a.memory_high_water() == own_a
        own_b, _ = bj.witness_slots_bytes_split(11, V, 1, 0, lookup=_lk(c))
        plan = nat.memory_plan_lanes(3)["total"]  # two lanes and the parent
        total = plan + hint_bytes + parent_bytes + own_a + own_b
        ctx.set_memory_limit(total - 1)
        high, launches = b.memory_high_water(), b.launch_count()
        h = ctypes.c_void_p()
        assert lib.bj_witness_slots_create(b._h, nat._h, 1, 0, ctypes.byref(h)) == OOM and not h.value
        msg = lib.bj_last_error(b._h).decode()
        for term in (plan, hint_bytes, parent_bytes, own_a, own_b, total, total - 1):
            assert str(term) in msg, (term, msg)
        assert b.memory_high_water() == high and b.launch_count() == launches
        ctx.set_memory_limit(total)
        set_b = nat.witness_slots(1, 0, ctx=b)
        assert b.memory_high_water() == own_b
        # a third lane: bj_ctx_create_lane adds the lanes' sets (not the parent's) to its check
        lanes3 = nat.memory_plan_lanes(4)["total"]
        ctx.set_memory_limit(lanes3 + own_a + own_b - 1)
        assert lib.bj_ctx_create_lane(ctx._h, ctypes.byref(h)) == OOM and not h.value
        assert str(own_a + own_b) in lib.bj_last_error(ctx._h).decode()
        ctx.set_memory_limit(lanes3 + own_a + own_b)
        third = ctx.lane()
        # freeing a set gives its bytes back
        set_a.close()
        ctx.set_memory_limit(nat.memory_plan_lanes(4)["total"] + hint_bytes + parent_bytes + own_b + own_a)
        nat.witness_slots(2, n_values, ctx=third).close()
        for s in (set_b, parent_set):
            s.close()
        for ln in (a, b, third):
            ln.close()
        nat.close()
    finally:
        ctx.close()


def test_lane_set_refusals(bj):
    lib = bj.native.lib
    cs = _witnesses(bj, "bench", 11)
    c, cfg = cs[0], _cfg("bench")
    V, n = c["variables"].shape
    hint, n_values = _vec_hint(V, n)
    v, m = bj.to_numpy(c["variables"]), bj.to_numpy(c["lookup"]["multiplicities"])
    ctx, other = bj.Context(0), bj.Context(0)
    try:
        nat, foreign = _setup(ctx, c, cfg), _setup(other, c, cfg)
        a, b = ctx.lane(), ctx.lane()
        h = ctypes.c_void_p()
        # a setup of another parent
        assert lib.bj_witness_slots_create(a._h, foreign._h, 1, 0, ctypes.byref(h)) == INVALID and not h.value
        assert b"another context" in lib.bj_last_error(a._h)
        set_a = nat.witness_slots(1, 0, ctx=a)
        set_p = nat.witness_slots(1, 0)
        set_a.upload(0, v, m)
        set_p.upload(0, v, m)
        counts = [x.launch_count() for x in (ctx, a, b)]
        p = ctypes.c_void_p()
        assert lib.bj_prove_slot(b._h, nat._h, set_a._h, 0, ctypes.byref(p)) == INVALID      # another lane's set
        assert lib.bj_prove_slot(ctx._h, nat._h, set_a._h, 0, ctypes.byref(p)) == INVALID    # a lane's set on the parent
        assert lib.bj_prove_slot(a._h, nat._h, set_p._h, 0, ctypes.byref(p)) == INVALID     # the parent's set on a lane
        assert not p.value
        # a hint replaced under a live lane set
        with pytest.raises(bj.BoojumError) as e:
            nat.attach_variables_hint(hint)
        assert e.value.status == INVALID and "lane" in str(e.value)
        # a lane destroyed under its live set: refused, and the lane stays usable
        assert lib.bj_ctx_destroy(a._h) == INVALID
        assert b"slot set" in lib.bj_last_error(a._h)
        assert [x.launch_count() for x in (ctx, a, b)] == counts
        want = nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True)
        assert set_a.prove(0) == want and set_p.prove(0) == want
        set_a.close()
        nat.attach_variables_hint(hint)  # no lane set alive any more
        a.close()
        b.close()
        set_p.close()
        nat.close()
        foreign.close()
    finally:
        ctx.close()
        other.close()
