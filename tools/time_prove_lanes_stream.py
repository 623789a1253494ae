"""Throughput of one setup proved from pinned host witnesses (proofs per second), as columns and as the reference's WitnessVec
(all_values + u32 multiplicities gathered through the setup's u32 copy hint), three ways:
  (a) one_by_one   bj_upload of the witness on the setup's context, then bj_prove, one after the other;
  (b) stream       NativeSetup.prove_stream over a 2-slot set of the setup's context (the next upload overlaps the proof);
  (c) lanes_N      N lanes of the setup's context (Context.lane), each streaming its share (witness i on lane i % N) through
                   its own 2-slot set on its own copy stream, from its own thread, for every N = 2, 3, 4 whose lanes and sets
                   fit (a lane or set the memory check refuses is reported as refused, not measured).
Every proof is checked equal to (a)'s proof of the same witness.  Each configuration of (b) and (c) is set up on its own,
alternated with (a) over --rounds rounds, and released again; the best round counts, for (a) over all its rounds.  The columns
configurations run first; then the hint is attached and the WitnessVec ones run.  For every lane count the pool high-water
mark of each lane is reported beside its planned part (bj_proof_memory_plan_lane_pool plus its set's own bytes).  Workloads:
the production shape at 2^20 (155 columns, Q = 8 over L = 2; Poseidon2 and Blake2s) and the bench shape at 2^16
(synthetic.generate with lookups, Q = 4 over L = 8).  The card's name and power limit are read at the start of the run.
Prints one JSON line per workload and writes them to --out."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_prove_concurrent import on_threads  # noqa: E402
from time_prove_stream import gpu_info, pinned, workload  # noqa: E402

OOM = -4  # BJ_ERR_OOM
SLOTS = 2


def run(bj, name, log_n, steps, rounds, distinct):
    import torch
    c, cfg, ws = workload(bj, name, log_n, distinct)
    V, n = ws[0][0].shape
    lk = dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"])
    order = [k % distinct for k in range(steps)]
    cols = [(pinned(v), pinned(m)) for v, m in ws]
    perm = np.random.default_rng(5).permutation(V * n).astype(np.uint64)
    vec = []
    for v, m in ws:
        av = np.empty(V * n, np.uint64)
        av[perm] = v.reshape(-1)
        vec.append((pinned(av), pinned(m.astype(np.uint32))))
    del ws

    lib = bj.native.lib
    ctx = bj.Context(0)
    nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                           public_inputs=c["public_inputs"])
    dv = torch.empty((V, n), dtype=torch.int64, device="cuda:0")
    dm = torch.empty(n, dtype=torch.int64, device="cuda:0")

    def one_by_one():
        out = []
        for k in order:
            v, m = cols[k]
            ctx._check(lib.bj_upload(ctx._h, ctx._ptr(dv), ctypes.c_void_p(v.data_ptr()), dv.numel() * 8))
            ctx._check(lib.bj_upload(ctx._h, ctx._ptr(dm), ctypes.c_void_p(m.data_ptr()), dm.numel() * 8))
            out.append(nat.prove(dv, dm, as_json=True))
        return out

    want = one_by_one()[:distinct]
    expected = [want[k] for k in order]
    res = dict(workload=name, rows_log2=log_n, columns=V, proofs=steps, distinct_witnesses=distinct, plan=nat.plan,
               slots_per_set=SLOTS, witness_bytes=(V + 1) * n * 8)
    seq_times = []

    def timed(kind, fn):
        """fn alternated with (a) over the rounds; the best round of fn is recorded, (a)'s times are kept"""
        ts = []
        for _ in range(rounds):
            for k, f in (("one_by_one", one_by_one), (kind, fn)):
                torch.cuda.synchronize()
                t = time.perf_counter()
                got = f()
                secs = time.perf_counter() - t
                assert got == expected, k
                (seq_times if k == "one_by_one" else ts).append(secs)
        res.setdefault(kind, {}).update(proofs_per_second=round(steps / min(ts), 3), seconds_per_proof=round(min(ts) / steps, 4),
                                        rounds_seconds=[round(x, 3) for x in ts])

    def lanes_stream(sets, inputs):
        N = len(sets)
        per = on_threads([[lambda k=k: list(nat.prove_stream([inputs[order[i]] for i in range(k, steps, N)], slots=sets[k]))]
                          for k in range(N)])
        got = [None] * steps
        for k in range(N):
            for i, p in zip(range(k, steps, N), per[k][0]):
                got[i] = p
        return got

    for mode, inputs, max_values in (("columns", cols, 0), ("vec", vec, V * n)):
        if mode == "vec":
            nat.attach_variables_hint(perm.reshape(V, n))  # before any lane set
        suffix = "" if mode == "columns" else "_vec"
        own, hint = bj.witness_slots_bytes_split(log_n, V, SLOTS, max_values, lookup=lk)
        mine = nat.witness_slots(SLOTS, max_values)
        timed("stream" + suffix, lambda: list(nat.prove_stream([inputs[k] for k in order], slots=mine)))
        mine.close()
        for N in (2, 3, 4):
            kind = "lanes_%d%s" % (N, suffix)
            mp = nat.memory_plan_lanes(N + 1)  # the parent counts as one proving context
            lanes, sets = [], []
            try:
                for _ in range(N):
                    lanes.append(ctx.lane())
                for ln in lanes:
                    sets.append(nat.witness_slots(SLOTS, max_values, ctx=ln))
            except bj.BoojumError as e:
                assert e.status == OOM, e
                res[kind] = dict(refused="not measured: %s" % e, plan_bytes_total=mp["total"], set_bytes_per_lane=own, hint_bytes=hint)
                for s in sets:
                    s.close()
                for ln in lanes:
                    ln.close()
                continue
            assert lanes_stream(sets, inputs) == expected  # warm-up
            res[kind] = dict(pool_high_water=[ln.memory_high_water() for ln in lanes], pool_plan_per_lane=mp["lane_pool"] + own,
                             plan_lane_pool=mp["lane_pool"], set_bytes_per_lane=own, hint_bytes=hint,
                             plan_bytes_per_lane=mp["lane"], plan_bytes_total=mp["total"])
            timed(kind, lambda sets=sets: lanes_stream(sets, inputs))
            for s in sets:
                s.close()
            for ln in lanes:
                ln.close()

    seq = min(seq_times)
    res["one_by_one"] = dict(proofs_per_second=round(steps / seq, 3), seconds_per_proof=round(seq / steps, 4),
                             rounds_seconds=[round(x, 3) for x in seq_times])
    for kind, r in res.items():
        if isinstance(r, dict) and "proofs_per_second" in r and kind != "one_by_one":
            r["speedup_over_one_by_one"] = round(seq / (r["seconds_per_proof"] * steps), 3)
    nat.close()
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12, help="proofs per timed case (a multiple of 2, 3 and 4)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=3, help="distinct pinned host witnesses, cycled over the steps")
    ap.add_argument("--workloads", default="production_poseidon2:20,production_blake2s:20,bench:16")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_prove_lanes_stream.json"))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "time_prove_lanes_stream needs a CUDA device"
    import era_boojum_b200 as bj
    info = gpu_info()
    lines = []
    for w in args.workloads.split(","):
        name, log_n = w.split(":")
        res = dict(run(bj, name, int(log_n), args.steps, args.rounds, args.distinct), **info)
        print(json.dumps(res), flush=True)
        lines.append(res)
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
