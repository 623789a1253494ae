"""Throughput of one setup proved several witnesses at a time on one GPU (proofs per second), four ways:
  (a) sequential       bj_prove on the setup's own context, one proof after the other;
  (b) parent_and_lane  the setup's context and one lane of it (Context.lane) proving at once from two host threads;
      lanes_N          N = 2, 3, 4 lanes of that context, each proving from its own host thread, all reading the one setup
                       (a configuration whose planned memory does not fit is reported as refused);
  (c) two_contexts     two independent contexts, each with its own setup of the same circuit, proving from two threads (where
                       a second whole plan fits on the device).
Witnesses are distinct and already on the device.  Every proof is checked equal to (a)'s proof of the same witness.  Each
configuration of (b) and (c) is set up on its own, alternated with (a) over --rounds rounds, and released again; the best
round counts, for (a) over all its rounds.  For every lane count the pool high-water mark of each fresh
lane is reported beside the lane part of bj_proof_memory_plan_lanes.  Workloads: the production shape at 2^20 (155 columns,
Q = 8 over L = 2; Poseidon2 and Blake2s) and the bench shape at 2^16 and 2^21 (synthetic.generate with lookups, Q = 4 over
L = 8).  Prints one JSON line per workload (and writes them to --out if given)."""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_prove_stream import gpu_info  # noqa: E402

OOM = -4  # BJ_ERR_OOM


def workload(bj, name, log_n, distinct):
    """(setup inputs, config, list of `distinct` device witnesses (variables, multiplicities))"""
    from era_boojum_b200 import prover, synthetic
    ctx = bj.Context(0)
    ws = []
    for k in range(distinct):
        if name.startswith("production"):
            c = synthetic.generate_production_shaped(ctx, log_n, seed=42, witness_seed=2000 + k)
            hasher = name.split("_")[1]
            cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100, hasher=hasher, transcript=hasher)
        else:
            v, s, cc, g, q, lk = synthetic.generate(ctx, log_n, 60, seed=42, lookup=True, witness_seed=2000 + k)
            c = dict(variables=v, sigmas=s, constants=cc, gates=g, quotient_degree=q, lookup=lk, public_inputs=[])
            cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)
        ws.append((c["variables"], c["lookup"]["multiplicities"]))
        setup_inputs = c
    ctx.synchronize()
    ctx.close()
    return setup_inputs, cfg, ws


def on_threads(jobs):
    """runs each job (a list of callables) on its own thread, all started together -> the results in job order"""
    out = [None] * len(jobs)
    errors = []
    start = threading.Barrier(len(jobs))

    def run(k):
        try:
            start.wait()
            out[k] = [f() for f in jobs[k]]
        except Exception as e:  # noqa: BLE001 - re-raised below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(k,)) for k in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    return out


def run(bj, name, log_n, steps, rounds, distinct):
    import torch
    c, cfg, ws = workload(bj, name, log_n, distinct)
    order = [k % distinct for k in range(steps)]

    def setup(ctx):
        return ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                                public_inputs=c["public_inputs"])

    ctx = bj.Context(0)
    nat = setup(ctx)
    want = [nat.prove(*w, as_json=True) for w in ws]

    def interleaved(proofs_by_job, n_jobs):
        """the proofs of `order` dealt round-robin to n_jobs jobs, back in order"""
        got = [None] * steps
        for j, ps in enumerate(proofs_by_job):
            for i, p in zip(range(j, steps, n_jobs), ps):
                got[i] = p
        return got

    res = dict(workload=name, rows_log2=log_n, columns=int(ws[0][0].shape[0]), proofs=steps, distinct_witnesses=distinct, plan=nat.plan)

    def sequential():
        return [nat.prove(*ws[k], as_json=True) for k in order]

    def dealt(provers):
        """the proofs of `order` dealt round-robin to the provers (callables of a witness), each on its own thread"""
        n = len(provers)
        return interleaved(on_threads([[lambda f=provers[j], i=i: f(ws[order[i]]) for i in range(j, steps, n)] for j in range(n)]), n)

    def on_lane(ln):
        return lambda w: nat.prove(*w, as_json=True, ctx=ln)

    def timed(kind, fn):
        """fn alternated with the sequential case over the rounds -> best seconds of fn; the sequential times are kept"""
        ts = []
        for _ in range(rounds):
            for k, f in (("sequential", sequential), (kind, fn)):
                torch.cuda.synchronize()
                t = time.perf_counter()
                got = f()
                secs = time.perf_counter() - t
                assert got == [want[i] for i in order], k
                (seq_times if k == "sequential" else ts).append(secs)
        res.setdefault(kind, {}).update(proofs_per_second=round(steps / min(ts), 3), seconds_per_proof=round(min(ts) / steps, 4),
                                        rounds_seconds=[round(x, 3) for x in ts])

    seq_times = []
    # one phase per configuration: its lanes (or second context) exist during that phase only.  parent_and_lane: the parent
    # and one lane proving at once (two proofs in flight); lanes_N: N lanes, the parent idle
    for kind, n_lanes, parent_proves in (("parent_and_lane", 1, True), ("lanes_2", 2, False), ("lanes_3", 3, False), ("lanes_4", 4, False)):
        mp = nat.memory_plan_lanes(n_lanes + 1)  # the parent counts as one proving context
        lanes = []
        try:
            for _ in range(n_lanes):
                lanes.append(ctx.lane())
        except bj.BoojumError as e:
            assert e.status == OOM, e
            for ln in lanes:
                ln.close()
            res[kind] = dict(refused="the setup and %d proving contexts plan %d bytes, above the limit the setup was planned under"
                             % (n_lanes + 1, mp["total"]))
            continue
        # warm-up: one proof per fresh lane, at the same time; then the pool high-water mark of each lane
        first = on_threads([[lambda ln=ln, k=k: nat.prove(*ws[k % distinct], as_json=True, ctx=ln)] for k, ln in enumerate(lanes)])
        assert [p[0] for p in first] == [want[k % distinct] for k in range(n_lanes)]
        res[kind] = dict(pool_high_water=[ln.memory_high_water() for ln in lanes], pool_plan_per_lane=mp["lane_pool"],
                         plan_bytes_per_lane=mp["lane"], plan_bytes_setup=mp["setup"], plan_bytes_total=mp["total"])
        provers = ([lambda w: nat.prove(*w, as_json=True)] if parent_proves else []) + [on_lane(ln) for ln in lanes]
        timed(kind, lambda provers=provers: dealt(provers))
        for ln in lanes:
            ln.close()

    plan = nat.memory_plan()
    whole = plan["pool"] + plan["outside_pool"]
    if 1.1 * whole < torch.cuda.mem_get_info(0)[0]:
        ctx2 = bj.Context(0)
        nat2 = setup(ctx2)
        assert nat2.prove(*ws[0], as_json=True) == want[0]
        timed("two_contexts", lambda: dealt([lambda w: nat.prove(*w, as_json=True), lambda w: nat2.prove(*w, as_json=True)]))
        nat2.close()
        ctx2.close()
    else:
        res["two_contexts"] = dict(refused="a second whole plan of %d bytes does not fit beside the first" % whole)

    for _ in range(rounds if not seq_times else 0):  # nothing else fitted: the sequential case alone
        torch.cuda.synchronize()
        t = time.perf_counter()
        assert sequential() == [want[i] for i in order]
        seq_times.append(time.perf_counter() - t)
    seq = min(seq_times)
    res["sequential"] = dict(proofs_per_second=round(steps / seq, 3), seconds_per_proof=round(seq / steps, 4),
                             rounds_seconds=[round(x, 3) for x in seq_times])
    for kind, r in res.items():
        if isinstance(r, dict) and "proofs_per_second" in r and kind != "sequential":
            r["speedup_over_sequential"] = round(seq / (r["seconds_per_proof"] * steps), 3)
    nat.close()
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12, help="proofs per timed case (a multiple of 2, 3 and 4)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=4, help="distinct device witnesses, cycled over the steps")
    ap.add_argument("--workloads", default="production_poseidon2:20,production_blake2s:20,bench:16,bench:21")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "time_prove_concurrent needs a CUDA device"
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
