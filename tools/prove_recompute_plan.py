"""Prove on the recompute plan (Context.allow_recompute_plan): one GPU, no coset of the setup, witness or stage-2 columns kept.
Prints one JSON line per workload, with the GPU name and power limit read in the same run:
- production: the production-shaped circuit (155 columns, 8 lookups of width 3, Q = 8 over L = 2, cap 32) at --compare-log-n,
  proved on the resident, streamed and recompute plans on the same inputs in alternating rounds; the proofs must be identical.
- bench: the bench circuit (60 columns, 8 lookups of width 4, Q = 4 over L = 8, cap 16) at --bench-log-n, the compact plan
  against the recompute plan (one after the other: both contexts' pools do not fit together); the proofs must be identical.
- production on the recompute plan alone at every --log-n: setup and proof seconds, pool high-water against the plan, verified
  by oracle/verifier.py.
Each plan runs under a limit equal to its own planned bytes.  --out also writes the lines to a file.
usage: prove_recompute_plan.py [--compare-log-n 20] [--bench-log-n 22] [--log-n 22 23] [--rounds 3] [--out FILE]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import era_boojum_b200 as bj  # noqa: E402
from era_boojum_b200 import prover, synthetic  # noqa: E402
from oracle import verifier as OV  # noqa: E402
from tools.prove_production_shape_limited import gpu_power_limit_w  # noqa: E402

PROD_CFG = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
BENCH_CFG = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)


class Run:
    """one context under a limit equal to `plan`'s bytes, its setup and its proofs"""

    def __init__(self, c, cfg, plan, limit):
        self.c = c
        self.ctx = bj.Context.on_current_stream(0)
        self.ctx.set_memory_limit(limit)
        self.ctx.allow_recompute_plan(plan == "recompute")
        self.ctx.memory_high_water(reset=True)
        t0 = time.perf_counter()
        self.nat = self.ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                                         public_inputs=c["public_inputs"])
        torch.cuda.synchronize()
        self.setup_s = time.perf_counter() - t0
        assert self.nat.plan == plan, (self.nat.plan, plan)
        self.seconds, self.stages = [], []
        self.first_s, self.proof = self.prove()
        self.high_water = self.ctx.memory_high_water()  # setup + first proof on a fresh context: the planned pool peak

    def prove(self):
        tm = {}
        t0 = time.perf_counter()
        proof = self.nat.prove(self.c["variables"], self.c["lookup"]["multiplicities"], timings=tm, as_json=True)
        dt = time.perf_counter() - t0
        self.stages.append(tm)
        return dt, proof

    def timed(self):
        dt, proof = self.prove()
        self.seconds.append(round(dt, 4))
        assert proof == self.proof, "a proof of the same inputs moved"

    def report(self):
        mp = self.nat.memory_plan()
        best = min(range(len(self.stages)), key=lambda i: sum(self.stages[i].values()))
        return {"planned_pool_peak_bytes": mp["pool"], "planned_outside_pool_bytes": mp["outside_pool"], "chunk": mp["chunk"],
                "pool_high_water_bytes": self.high_water, "high_water_equals_plan": self.high_water == mp["pool"],
                "setup_seconds": round(self.setup_s, 3), "first_prove_seconds": round(self.first_s, 3), "prove_seconds": self.seconds,
                "stage_seconds": {k: round(v, 4) for k, v in self.stages[best].items()}}

    def close(self):
        self.nat.close()
        self.ctx.synchronize()
        self.ctx.close()


def production(log_n):
    gen = bj.Context.on_current_stream(0)
    c = synthetic.generate_production_shaped(gen, log_n, seed=42)
    torch.cuda.synchronize()
    gen.close()
    torch.cuda.empty_cache()
    return c


def bench_circuit(log_n):
    gen = bj.Context.on_current_stream(0)
    v, s, k, g, q, lk = synthetic.generate(gen, log_n, 60, seed=42, lookup=True)
    torch.cuda.synchronize()
    gen.close()
    torch.cuda.empty_cache()
    return dict(variables=v, sigmas=s, constants=k, gates=g, quotient_degree=q, lookup=lk, public_inputs=[])


def plan_of(c, log_n, cfg):
    lk = dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"])
    return bj.proof_memory_plan(log_n, c["sigmas"].shape[0], c["constants"].shape[0], c["quotient_degree"], cfg, lookup=lk)


def verify(run):
    t0 = time.perf_counter()
    ok = bool(OV.verify(run.nat.vk(), json.loads(run.proof)))
    return ok, round(time.perf_counter() - t0, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare-log-n", type=int, nargs="*", default=[20])
    ap.add_argument("--bench-log-n", type=int, nargs="*", default=[22])
    ap.add_argument("--log-n", type=int, nargs="*", default=[22, 23])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    head = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": gpu_power_limit_w()}
    lines = []

    def emit(out):
        line = json.dumps(dict(head, **out))
        print(line, flush=True)
        lines.append(line)
        if args.out:
            with open(args.out, "w") as f:
                f.write("\n".join(lines) + "\n")

    for log_n in args.compare_log_n:
        c = production(log_n)
        plan = plan_of(c, log_n, PROD_CFG)
        runs = {"resident": Run(c, PROD_CFG, "resident", plan["resident"]), "streamed": Run(c, PROD_CFG, "streamed", plan["streamed"]),
                "recompute": Run(c, PROD_CFG, "recompute", plan["recompute"])}
        for _ in range(args.rounds):  # alternating, so that every plan sees the same state of a shared device
            for r in runs.values():
                r.timed()
        out = {"workload": "production-shaped circuit 2^%d x 155 columns, Q = 8 over L = 2, cap 32, poseidon2: resident, streamed and "
               "recompute plans alternated" % log_n, "planned_bytes": plan,
               "identical": len({r.proof for r in runs.values()}) == 1}
        out["verified"], out["verify_cpu_seconds"] = verify(runs["recompute"])
        for name, r in runs.items():
            out[name] = r.report()
            r.close()
        del c
        torch.cuda.empty_cache()
        emit(out)
        assert out["identical"] and out["verified"]

    for log_n in args.bench_log_n:
        c = bench_circuit(log_n)
        plan = plan_of(c, log_n, BENCH_CFG)
        out = {"workload": "bench circuit 2^%d x 60 columns, Q = 4 over L = 8, cap 16, poseidon2: compact, then recompute plan" % log_n,
               "planned_bytes": plan}
        proofs = {}
        for name in ("compact", "recompute"):
            r = Run(c, BENCH_CFG, name, plan[name])
            for _ in range(args.rounds):
                r.timed()
            out[name] = r.report()
            proofs[name] = r.proof
            if name == "recompute":
                out["verified"], out["verify_cpu_seconds"] = verify(r)
            r.close()
            torch.cuda.empty_cache()
        out["identical"] = proofs["compact"] == proofs["recompute"]
        del c
        torch.cuda.empty_cache()
        emit(out)
        assert out["identical"] and out["verified"]

    for log_n in args.log_n:
        c = production(log_n)
        plan = plan_of(c, log_n, PROD_CFG)
        inputs = sum(t.numel() * 8 for t in (c["variables"], c["sigmas"], c["constants"], c["lookup"]["tables"], c["lookup"]["multiplicities"]))
        r = Run(c, PROD_CFG, "recompute", plan["recompute"])
        for _ in range(max(1, args.rounds - 1)):
            r.timed()
        out = {"workload": "production-shaped circuit 2^%d x 155 columns, Q = 8 over L = 2, cap 32, poseidon2: recompute plan" % log_n,
               "planned_bytes": plan, "input_bytes": inputs, "recompute": r.report()}
        out["verified"], out["verify_cpu_seconds"] = verify(r)
        r.close()
        del c
        torch.cuda.empty_cache()
        emit(out)
        assert out["verified"] and out["recompute"]["high_water_equals_plan"]


if __name__ == "__main__":
    main()
