"""Repeated proving against one setup: witness slot sets (bj_witness_slots_*, bj_witness_upload(_vec), bj_prove_slot) and
NativeSetup.prove_stream.  Several pairwise different witnesses of ONE setup (same sigmas, constants and tables: the synthetic
generators with the circuit seed fixed and the witness seed varied) are streamed through 1, 2 and 4 slots, from pinned and
pageable host memory, as columns and as the reference's WitnessVec (all_values + u32 multiplicities gathered through the
setup's copy hint), on the resident, compact and streamed memory plans and on sharded contexts.  Every streamed proof must be
byte for byte the proof bj_prove gives on the same witness uploaded with bj_upload, which the verifier accepts."""
import ctypes
import json
import threading

import numpy as np
import pytest

from oracle import verifier as OV

pytestmark = pytest.mark.gpu

INVALID, OOM = -1, -4  # BJ_ERR_INVALID_ARG, BJ_ERR_OOM
K = 3                  # witnesses per setup


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


def _witnesses(bj, shape, log_n, k=K):
    """k circuits of one structure and k witness seeds -> list of dicts (device tensors); the setup inputs are checked equal"""
    import torch
    from era_boojum_b200 import synthetic
    ctx = bj.Context(0)
    out = []
    for ws in range(k):
        if shape == "production":
            out.append(synthetic.generate_production_shaped(ctx, log_n, seed=90 + log_n, witness_seed=500 + ws))
        else:
            v, s, c, g, q, lk = synthetic.generate(ctx, log_n, 60, seed=30 + log_n, lookup=True, witness_seed=600 + ws)
            out.append(dict(variables=v, sigmas=s, constants=c, gates=g, quotient_degree=q, lookup=lk, public_inputs=[(3, 5)]))
    ctx.synchronize()
    ctx.close()
    for c in out[1:]:
        assert torch.equal(c["sigmas"], out[0]["sigmas"]) and torch.equal(c["constants"], out[0]["constants"])
        assert torch.equal(c["lookup"]["tables"], out[0]["lookup"]["tables"])
    for i in range(k):
        for j in range(i):
            assert not torch.equal(out[i]["variables"], out[j]["variables"])
    return out


def _cfg(shape, hasher="poseidon2"):
    from era_boojum_b200 import prover
    if shape == "production":
        return prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100, hasher=hasher, transcript=hasher)
    return prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100, hasher=hasher, transcript=hasher)


def _setup(ctx, c, cfg):
    return ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                            public_inputs=c["public_inputs"])


def _host(bj, c):
    """(variables [V, n], multiplicities [n]) as pageable numpy uint64"""
    return bj.to_numpy(c["variables"]), bj.to_numpy(c["lookup"]["multiplicities"])


def _pinned(a):
    """a pinned host copy (torch, same bits) of a uint64 or uint32 array"""
    import torch
    signed = {8: (np.int64, torch.int64), 4: (np.int32, torch.int32)}[a.dtype.itemsize]
    t = torch.empty(a.shape, dtype=signed[1], pin_memory=True)
    t.copy_(torch.from_numpy(np.ascontiguousarray(a).view(signed[0])))
    assert t.is_pinned()
    return t


def _vec_hint(V, n, extra=5, seed=7):
    """a DenseVariablesCopyHint of one setup: cell (c, row) reads all_values[perm[c * n + row]]"""
    perm = np.random.default_rng(seed).permutation(V * n + extra)[: V * n]
    return perm.reshape(V, n).astype(np.uint64), V * n + extra


def _vec(variables, multiplicities, hint, n_values):
    """the WitnessVec of a witness under `hint`: all_values (u64) and the multiplicities as u32"""
    av = np.full(n_values, 12345, np.uint64)
    av[hint.reshape(-1)] = variables.reshape(-1)
    return av, multiplicities.astype(np.uint32)


_REFERENCE = {}


def _one_by_one(bj, shape, log_n):
    """(circuits, proofs of bj_prove on each witness uploaded with bj_upload, vk) - the proofs checked by the verifier"""
    key = (shape, log_n)
    if key in _REFERENCE:
        return _REFERENCE[key]
    import torch
    cs = _witnesses(bj, shape, log_n)
    ctx = bj.Context(0)
    nat = _setup(ctx, cs[0], _cfg(shape))
    proofs = []
    for c in cs:
        v, m = _host(bj, c)
        dv = torch.empty(v.shape, dtype=torch.int64, device="cuda:0")
        dm = torch.empty(m.shape, dtype=torch.int64, device="cuda:0")
        lib = bj.native.lib
        ctx._check(lib.bj_upload(ctx._h, ctx._ptr(dv), v.ctypes.data_as(ctypes.c_void_p), v.nbytes))
        ctx._check(lib.bj_upload(ctx._h, ctx._ptr(dm), m.ctypes.data_as(ctypes.c_void_p), m.nbytes))
        proofs.append(nat.prove(dv, dm, as_json=True))
    vk = nat.vk()
    nat.close()
    ctx.close()
    for p in proofs:
        assert OV.verify(vk, json.loads(p))
    assert len(set(proofs)) == len(proofs)
    _REFERENCE[key] = (cs, proofs, vk)
    return _REFERENCE[key]


def _slot_bytes(bj, c, n_slots, max_values):
    V, n = c["variables"].shape
    return bj.witness_slots_bytes(n.bit_length() - 1, V, n_slots, max_values, lookup=c["lookup"])


def _inputs(bj, cs, memory, mode, hint, n_values):
    out = []
    for c in cs:
        v, m = _host(bj, c)
        if mode == "vec":
            v, m = _vec(v, m, hint, n_values)
        out.append((_pinned(v), _pinned(m)) if memory == "pinned" else (v, m))
    return out


@pytest.mark.parametrize("plan,n_slots,memory,mode", [
    ("resident", 1, "pageable", "columns"),
    ("resident", 2, "pinned", "columns"),
    ("resident", 4, "pageable", "vec"),
    ("resident", 2, "pinned", "vec"),
    ("compact", 2, "pinned", "columns"),
    ("compact", 2, "pageable", "vec"),
    ("streamed", 2, "pageable", "columns"),
    ("streamed", 1, "pinned", "vec"),
    ("streamed", 4, "pinned", "columns")])
def test_stream_equals_one_by_one(bj, plan, n_slots, memory, mode):
    shape = "production" if plan == "streamed" else "bench"
    cs, want, _ = _one_by_one(bj, shape, 10)
    V, n = cs[0]["variables"].shape
    hint, n_values = _vec_hint(V, n)
    max_values = n_values if mode == "vec" else 0
    slots_bytes = _slot_bytes(bj, cs[0], n_slots, max_values)
    ctx = bj.Context(0)
    try:
        if plan != "resident":
            lk = dict(width=cs[0]["lookup"]["width"], num_repetitions=cs[0]["lookup"]["num_repetitions"])
            mp = bj.proof_memory_plan(10, V, cs[0]["constants"].shape[0], cs[0]["quotient_degree"], _cfg(shape), lookup=lk)
            # the compact plan widens its recompute chunk into up to half the headroom: twice the slot bytes keep the slots in
            ctx.set_memory_limit(mp[plan] + 2 * slots_bytes)
        nat = _setup(ctx, cs[0], _cfg(shape))
        assert nat.plan == plan
        if mode == "vec":
            nat.attach_variables_hint(hint)
        slots = nat.witness_slots(n_slots, max_values)
        got = list(nat.prove_stream(_inputs(bj, cs, memory, mode, hint, n_values), slots=slots))
        assert got == want
        high = ctx.memory_high_water()
        assert high <= nat.memory_plan()["pool"] + slots_bytes, (high, nat.memory_plan(), slots_bytes)
        slots.close()
        nat.close()
    finally:
        ctx.close()


def test_default_stream_and_order(bj):
    """prove_stream with its own 2-slot set; swapping two witnesses swaps their proofs; re-uploads into a slot whose proof just
    returned, and two uploads into one slot before its proof, give the right proofs"""
    cs, want, _ = _one_by_one(bj, "bench", 10)
    ctx = bj.Context(0)
    try:
        nat = _setup(ctx, cs[0], _cfg("bench"))
        hw = [_host(bj, c) for c in cs]
        assert list(nat.prove_stream(hw)) == want
        assert list(nat.prove_stream([hw[1], hw[0], hw[2]])) == [want[1], want[0], want[2]]
        order = [0, 1, 2, 0, 2, 1, 1]
        assert list(nat.prove_stream([hw[i] for i in order], slots=nat.witness_slots(2))) == [want[i] for i in order]
        one = nat.witness_slots(1)
        for i in (2, 0, 1):
            one.upload(0, *hw[i])
            assert one.prove(0) == want[i]
        pinned = [(_pinned(v), _pinned(m)) for v, m in hw]
        one.upload(0, *pinned[2])
        one.upload(0, *pinned[1])
        assert one.prove(0) == want[1]
        one.close()
        nat.close()
    finally:
        ctx.close()


def test_device_gather_equals_materialize_columns(bj):
    """the u32 gather of bj_witness_upload_vec gives bj_materialize_columns' columns from the u64 hint: placeholders and rows past
    hint_rows are zero, non-canonical values are reduced; u32 multiplicities are widened and zero-padded to n"""
    cs, _, _ = _one_by_one(bj, "bench", 10)
    c = cs[0]
    V, n = c["variables"].shape
    rng = np.random.default_rng(3)
    hint_rows, n_values = n - 37, 5000
    hint = rng.integers(0, n_values, (V, hint_rows)).astype(np.uint64)
    hint[rng.random((V, hint_rows)) < 0.2] = np.uint64(1 << 63)
    values = rng.integers(0, 1 << 64, n_values, dtype=np.uint64)
    values[:3] = [bj.P, bj.P + 9, (1 << 64) - 1]
    hint[0, :3] = [0, 1, 2]
    mult = rng.integers(0, 1 << 32, n - 100, dtype=np.uint64).astype(np.uint32)
    ctx = bj.Context(0)
    try:
        nat = _setup(ctx, c, _cfg("bench"))
        nat.attach_variables_hint(hint)
        slots = nat.witness_slots(2, n_values)
        slots.upload_vec(1, values, mult)
        got_v, got_m = slots.columns(1)
        want_v = bj.to_numpy(ctx.materialize_variables_polynomials_from_dense_hint(bj.to_device(values), bj.to_device(hint), 10))
        assert np.array_equal(got_v, want_v)
        assert np.array_equal(got_m, np.concatenate([mult.astype(np.uint64), np.zeros(100, np.uint64)]))
        slots.close()
        nat.close()
    finally:
        ctx.close()


def test_slot_memory_limit(bj):
    """a limit one byte below the chosen plan + the slot bytes is refused with BJ_ERR_OOM, naming both, before any launch"""
    cs, _, _ = _one_by_one(bj, "bench", 10)
    ctx = bj.Context(0)
    try:
        nat = _setup(ctx, cs[0], _cfg("bench"))
        mp = nat.memory_plan()
        chosen = mp["pool"] + mp["outside_pool"]
        b = _slot_bytes(bj, cs[0], 2, 4096)
        ctx.set_memory_limit(chosen + b - 1)
        before = ctx.launch_count()
        with pytest.raises(bj.BoojumError) as e:
            nat.witness_slots(2, 4096)
        assert e.value.status == OOM and str(chosen) in str(e.value) and str(b) in str(e.value)
        assert ctx.launch_count() == before
        ctx.set_memory_limit(chosen + b)
        nat.witness_slots(2, 4096).close()
        nat.close()
    finally:
        ctx.close()


def test_argument_errors(bj):
    cs, _, _ = _one_by_one(bj, "bench", 10)
    v, m = _host(bj, cs[0])
    V, n = v.shape
    hint, n_values = _vec_hint(V, n)
    av, m32 = _vec(v, m, hint, n_values)
    lib = bj.native.lib
    ctx, other = bj.Context(0), bj.Context(0)
    try:
        a, b = _setup(ctx, cs[0], _cfg("bench")), _setup(ctx, cs[0], _cfg("bench"))
        x = _setup(other, cs[0], _cfg("bench"))
        before = ctx.launch_count()

        def refused(fn, *args):
            with pytest.raises(bj.BoojumError) as e:
                fn(*args)
            assert e.value.status == INVALID, e.value

        h = ctypes.c_void_p()
        assert lib.bj_witness_slots_create(ctx._h, x._h, 2, 0, ctypes.byref(h)) == INVALID      # another context's setup
        refused(a.witness_slots, 0)
        refused(a.witness_slots, 5)
        s = a.witness_slots(2)
        refused(s.upload, 2, v, m)                                                               # slot out of range
        refused(s.upload, 0, v, None)                                                            # lookup without multiplicities
        refused(s.prove, 1)                                                                      # never uploaded
        refused(s.prove, 7)
        refused(s.upload_vec, 0, av, m32)                                                        # no hint
        a.attach_variables_hint(hint)
        refused(s.upload_vec, 0, av, m32)                                                        # no all_values buffer
        sv = a.witness_slots(1, n_values)
        refused(sv.upload_vec, 0, av, None)                                                      # lookup without multiplicities
        refused(sv.upload_vec, 0, av[: n_values - 6], m32)                                       # fewer values than the hint names
        refused(sv.upload_vec, 0, np.zeros(n_values + 1, np.uint64), m32)                        # more than max_values
        s.upload(0, v, m)
        p = ctypes.c_void_p()
        assert lib.bj_prove_slot(ctx._h, b._h, s._h, 0, ctypes.byref(p)) == INVALID              # another setup's slots
        assert "another setup" in lib.bj_last_error(ctx._h).decode()
        assert ctx.launch_count() == before
        bad = np.array([[1 << 32] + [0] * (n - 1)] * V, np.uint64)
        refused(b.attach_variables_hint, bad)                                                    # index >= 2^32 - 1
        sv.close()
        s.close()
        for t in (a, b, x):
            t.close()
    finally:
        ctx.close()
        other.close()


@pytest.mark.parametrize("world,mode", [(2, "columns"), (4, "vec")])
def test_sharded_stream_equals_single_gpu(bj, world, mode):
    """production shape at 2^12 on thread ranks of the local transport (world 2: coset shard, 4: split shard): every rank
    uploads the same witnesses into its own slot set, and every rank's streamed proofs are the single-GPU proofs"""
    cs, want, _ = _one_by_one(bj, "production", 12)
    cfg = _cfg("production")
    V, n = cs[0]["variables"].shape
    hint, n_values = _vec_hint(V, n)
    group = bj.Comm.local_group(world)
    out, errs = [None] * world, []

    def run(rank):
        try:
            ctx = bj.Context(0)
            comm = bj.Comm.local(ctx, group, rank, world, cfg.fri_lde_factor)
            nat = _setup(ctx, cs[0], cfg)
            if mode == "vec":
                nat.attach_variables_hint(hint)
            out[rank] = list(nat.prove_stream(_inputs(bj, cs, "pinned", mode, hint, n_values)))
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
    bj.Comm.destroy_local_group(group)
    for rank in range(world):
        assert out[rank] == want, rank
