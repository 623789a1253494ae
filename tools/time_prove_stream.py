"""Times repeated proving against one setup from host witnesses, three ways:
  (a) one_by_one   bj_upload of the witness on the context's stream, then bj_prove (NativeSetup.prove), one after the other;
  (b) stream       NativeSetup.prove_stream over a 2-slot set, columns: witness k+1 is copied on the copy stream while
                   witness k is proved;
  (c) stream_vec   the same with the reference's WitnessVec (all_values + u32 multiplicities) gathered through the setup's
                   u32 copy hint.
Host witnesses are pinned (the copy engine reads them directly); `upload_seconds` is one witness's bj_upload alone (pinned and
pageable).  (a) and (b) are alternated over --rounds rounds.  Every proof of (b) and (c) is checked equal to (a)'s.
Workloads: the production shape at 2^20 (155 columns, Q = 8 over L = 2; Poseidon2 and Blake2s) and the bench shape at 2^21
(synthetic.generate with lookups, Q = 4 over L = 8).  Prints one JSON line per workload (and writes them to --out if given)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # the measurement stands without it, but says so
        return dict(gpu="unknown (%s)" % e)


def pinned(a):
    import torch
    signed = {8: (np.int64, torch.int64), 4: (np.int32, torch.int32)}[a.dtype.itemsize]
    t = torch.empty(a.shape, dtype=signed[1], pin_memory=True)
    t.copy_(torch.from_numpy(np.ascontiguousarray(a).view(signed[0])))
    return t


def workload(bj, name, log_n, distinct):
    """(setup inputs, config, list of `distinct` host witnesses (variables, multiplicities) as numpy uint64)"""
    from era_boojum_b200 import prover, synthetic
    ctx = bj.Context(0)
    ws = []
    for k in range(distinct):
        if name.startswith("production"):
            c = synthetic.generate_production_shaped(ctx, log_n, seed=42, witness_seed=1000 + k)
            hasher = name.split("_")[1]
            cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100, hasher=hasher, transcript=hasher)
        else:
            v, s, cc, g, q, lk = synthetic.generate(ctx, log_n, 60, seed=42, lookup=True, witness_seed=1000 + k)
            c = dict(variables=v, sigmas=s, constants=cc, gates=g, quotient_degree=q, lookup=lk, public_inputs=[])
            cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)
        ws.append((bj.to_numpy(c["variables"]), bj.to_numpy(c["lookup"]["multiplicities"])))
        del c["variables"]
        c["lookup"] = dict(c["lookup"], multiplicities=None)
        setup_inputs = c
    ctx.synchronize()
    ctx.close()
    return setup_inputs, cfg, ws


def run(bj, name, log_n, steps, rounds, distinct):
    import torch
    c, cfg, ws = workload(bj, name, log_n, distinct)
    V, n = ws[0][0].shape
    order = [k % distinct for k in range(steps)]
    pin = [(pinned(v), pinned(m)) for v, m in ws]
    lib = bj.native.lib
    import ctypes
    ctx = bj.Context(0)
    nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                           public_inputs=c["public_inputs"])
    dv = torch.empty((V, n), dtype=torch.int64, device="cuda:0")
    dm = torch.empty(n, dtype=torch.int64, device="cuda:0")

    def upload(v, m):
        ctx._check(lib.bj_upload(ctx._h, ctx._ptr(dv), ctypes.c_void_p(v.data_ptr() if hasattr(v, "data_ptr") else v.ctypes.data), dv.numel() * 8))
        ctx._check(lib.bj_upload(ctx._h, ctx._ptr(dm), ctypes.c_void_p(m.data_ptr() if hasattr(m, "data_ptr") else m.ctypes.data), dm.numel() * 8))

    def one_by_one():
        out = []
        for k in order:
            upload(*pin[k])
            out.append(nat.prove(dv, dm, as_json=True))
        return out

    slots = nat.witness_slots(2)

    def stream():
        return list(nat.prove_stream([pin[k] for k in order], slots=slots))

    # warm-up of every path, and the reference proofs
    want = [None] * distinct
    for k in range(distinct):
        upload(*pin[k])
        want[k] = nat.prove(dv, dm, as_json=True)
    assert stream() == [want[k] for k in order]
    ctx.synchronize()

    up = {}
    for kind, src in (("pinned", pin[0]), ("pageable", ws[0])):
        ctx.synchronize()
        t = time.perf_counter()
        for _ in range(3):
            upload(*src)
        ctx.synchronize()
        up[kind] = round((time.perf_counter() - t) / 3, 4)

    times = {"one_by_one": [], "stream": []}
    for _ in range(rounds):
        for kind, fn in (("one_by_one", one_by_one), ("stream", stream)):
            ctx.synchronize()
            if kind == "stream":
                ctx.memory_high_water(reset=True)
            t = time.perf_counter()
            got = fn()
            secs = time.perf_counter() - t
            assert got == [want[k] for k in order], kind
            times[kind].append(secs)
    high_stream = ctx.memory_high_water()
    slots.close()

    # (c) WitnessVec: all_values through a hint that scatters the cells (a permutation), u32 multiplicities
    perm = np.random.default_rng(5).permutation(V * n).astype(np.uint64)
    nat.attach_variables_hint(perm.reshape(V, n))
    vec = []
    for v, m in ws:
        av = np.empty(V * n, np.uint64)
        av[perm] = v.reshape(-1)
        vec.append((pinned(av), pinned(m.astype(np.uint32))))
    vslots = nat.witness_slots(2, V * n)
    assert list(nat.prove_stream([vec[k] for k in order], slots=vslots)) == [want[k] for k in order]
    times["stream_vec"] = []
    ctx.memory_high_water(reset=True)
    for _ in range(rounds):
        ctx.synchronize()
        t = time.perf_counter()
        got = list(nat.prove_stream([vec[k] for k in order], slots=vslots))
        times["stream_vec"].append(time.perf_counter() - t)
        assert got == [want[k] for k in order]
    high_vec = ctx.memory_high_water()
    mp = nat.memory_plan()
    lk = dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"])
    res = dict(workload=name, rows_log2=log_n, columns=V, proofs=steps, distinct_witnesses=distinct, plan=nat.plan,
               witness_bytes=(V + 1) * n * 8, upload_seconds=up, pool_plan_bytes=mp["pool"],
               slot_bytes=bj.witness_slots_bytes(log_n, V, 2, 0, lookup=lk), slot_bytes_vec=bj.witness_slots_bytes(log_n, V, 2, V * n, lookup=lk),
               pool_high_water_stream=high_stream, pool_high_water_stream_vec=high_vec)
    for kind, ts in times.items():
        best = min(ts)
        res[kind] = dict(proofs_per_second=round(steps / best, 3), seconds_per_proof=round(best / steps, 4),
                         rounds_seconds=[round(x, 3) for x in ts])
    res["stream_speedup"] = round(min(times["one_by_one"]) / min(times["stream"]), 3)
    vslots.close()
    nat.close()
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=4, help="distinct witnesses, cycled over the steps (host memory)")
    ap.add_argument("--workloads", default="production_poseidon2:20,production_blake2s:20,bench:21")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "time_prove_stream needs a CUDA device"
    import era_boojum_b200 as bj
    info = gpu_info()
    lines = []
    for w in args.workloads.split(","):
        name, log_n = w.split(":")
        res = dict(run(bj, name, int(log_n), args.steps, args.rounds, args.distinct), **info)
        print(json.dumps(res), flush=True)
        lines.append(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
