"""Prove on the one-GPU recompute plan with every coset cut into B row blocks (Context.set_max_row_blocks) and print one JSON line
per workload, with the GPU name and power limit read in the same run:
- compare: the production-shaped circuit (155 columns, 8 lookups of width 3, Q = 8 over L = 2, cap 32, Poseidon2) at
  --compare-log-n with B = 1, 2, 4 and 8 on the same inputs, each under a limit of its own plan, the four alternated over
  --rounds rounds: per-stage seconds, pool high-water against the plan; the proofs must be identical and verify.
- limited: the production shape at each --log-n under a limit of the plan at 2 row blocks (below the plan at 1), with up to 8
  allowed: setup and proof seconds, the row blocks chosen, pool high-water against the plan; the proof must verify.
- by the plan: for each --plan-log-n, the plan at every B and the natural-order inputs; the workload above runs there only if
  the smallest plan and the inputs fit the device's free memory, otherwise the line says "not run".
- kernels: for each --profile-log-n, one proof per B (after an untimed one) under torch.profiler, device time summed over the
  row-block fold kernel, the NTT kernels (forward and inverse share them) and everything else: where the extra time of B > 1
  goes.  A run of its own, so that tracing does not slow the timed workloads.
--out also writes the lines to a file.
usage: prove_recompute_blocks.py [--compare-log-n 20] [--log-n 23] [--plan-log-n 24] [--profile-log-n] [--rounds 3] [--out FILE]"""
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

CFG = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
BLOCKS = (1, 2, 4, 8)
V, C, Q, LOOKUP = 155, 8, 8, dict(width=3, num_repetitions=8)


def plans(log_n):
    return {B: bj.proof_memory_plan_recompute_blocks(log_n, V, C, Q, CFG, B, lookup=LOOKUP) for B in BLOCKS}


def input_bytes(log_n):
    """the natural-order inputs: variables and sigmas (155 each), 8 constants, 4 tables, the multiplicities"""
    return 8 * (1 << log_n) * (V + V + C + (LOOKUP["width"] + 1) + 1)


class Run:
    """one context on the recompute plan with up to `max_blocks` row blocks under `limit`, its setup and its proofs"""

    def __init__(self, c, max_blocks, limit):
        self.c = c
        self.ctx = bj.Context.on_current_stream(0)
        self.ctx.set_memory_limit(limit)
        self.ctx.allow_recompute_plan(True)
        self.ctx.set_max_row_blocks(max_blocks)
        self.ctx.memory_high_water(reset=True)
        t0 = time.perf_counter()
        self.nat = self.ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], CFG, lookup=c["lookup"],
                                         public_inputs=c["public_inputs"])
        torch.cuda.synchronize()
        self.setup_s = time.perf_counter() - t0
        assert self.nat.plan == "recompute", self.nat.plan
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
        return {"row_blocks": self.nat.row_blocks, "planned_pool_peak_bytes": mp["pool"], "planned_outside_pool_bytes": mp["outside_pool"],
                "chunk": mp["chunk"], "pool_high_water_bytes": self.high_water, "high_water_equals_plan": self.high_water == mp["pool"],
                "setup_seconds": round(self.setup_s, 3), "first_prove_seconds": round(self.first_s, 3), "prove_seconds": self.seconds,
                "stage_seconds": {k: round(v, 4) for k, v in self.stages[best].items()}}

    def verify(self):
        t0 = time.perf_counter()
        ok = bool(OV.verify(self.nat.vk(), json.loads(self.proof)))
        return ok, round(time.perf_counter() - t0, 2)

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


def limited(log_n, emit, rounds):
    p = plans(log_n)
    c = production(log_n)
    r = Run(c, 8, p[2])
    for _ in range(max(1, rounds - 1)):
        r.timed()
    out = {"workload": "production-shaped circuit 2^%d x 155 columns, Q = 8 over L = 2, cap 32, poseidon2: recompute plan under a "
           "limit of the plan at 2 row blocks, up to 8 allowed" % log_n, "planned_bytes_by_row_blocks": p,
           "input_bytes": input_bytes(log_n), "limit_bytes": p[2], "recompute": r.report()}
    out["verified"], out["verify_cpu_seconds"] = r.verify()
    r.close()
    del c
    torch.cuda.empty_cache()
    emit(out)
    assert out["verified"] and out["recompute"]["high_water_equals_plan"] and out["recompute"]["row_blocks"] == 2


def kernel_seconds(log_n, emit):
    from torch.profiler import ProfilerActivity, profile
    p = plans(log_n)
    c = production(log_n)
    out = {"workload": "production-shaped circuit 2^%d x 155 columns, Q = 8 over L = 2, cap 32, poseidon2: device time of one proof "
           "by kernel group under torch.profiler, recompute plan at 1, 2, 4 and 8 row blocks" % log_n}
    for B in BLOCKS:
        r = Run(c, B, p[B])
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            r.prove()
            torch.cuda.synchronize()
        groups = {"fold": 0.0, "ntt": 0.0, "other": 0.0}
        for ev in prof.key_averages():
            us = getattr(ev, "device_time_total", None)
            us = ev.cuda_time_total if us is None else us
            if not us:
                continue
            g = "fold" if "lde_unit_fold" in ev.key else "ntt" if "ntt_" in ev.key else "other"
            groups[g] += us / 1e6
        out["row_blocks_%d" % B] = {"row_blocks": r.nat.row_blocks, "kernel_seconds": {k: round(v, 4) for k, v in groups.items()}}
        r.close()
        torch.cuda.empty_cache()
    del c
    torch.cuda.empty_cache()
    emit(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare-log-n", type=int, nargs="*", default=[20])
    ap.add_argument("--log-n", type=int, nargs="*", default=[23])
    ap.add_argument("--plan-log-n", type=int, nargs="*", default=[24])
    ap.add_argument("--profile-log-n", type=int, nargs="*", default=[])
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
        p = plans(log_n)
        assert all(p[a] > p[b] for a, b in zip(BLOCKS, BLOCKS[1:])), p
        c = production(log_n)
        runs = {B: Run(c, B, p[B]) for B in BLOCKS}
        for _ in range(args.rounds):  # alternating, so that every B sees the same state of a shared device
            for r in runs.values():
                r.timed()
        out = {"workload": "production-shaped circuit 2^%d x 155 columns, Q = 8 over L = 2, cap 32, poseidon2: recompute plan at "
               "1, 2, 4 and 8 row blocks alternated" % log_n, "planned_bytes_by_row_blocks": p,
               "identical": len({r.proof for r in runs.values()}) == 1}
        out["verified"], out["verify_cpu_seconds"] = runs[8].verify()
        for B, r in runs.items():
            out["row_blocks_%d" % B] = r.report()
            r.close()
        del c
        torch.cuda.empty_cache()
        emit(out)
        assert out["identical"] and out["verified"]
        assert all(out["row_blocks_%d" % B]["row_blocks"] == B and out["row_blocks_%d" % B]["high_water_equals_plan"] for B in BLOCKS)

    for log_n in args.log_n:
        limited(log_n, emit, args.rounds)

    for log_n in args.plan_log_n:
        p = plans(log_n)
        free, total = torch.cuda.mem_get_info(0)
        need = min(p.values()) + input_bytes(log_n)
        if need <= free:
            limited(log_n, emit, args.rounds)
        else:
            emit({"workload": "production-shaped circuit 2^%d x 155 columns, Q = 8 over L = 2, cap 32: by the plan" % log_n,
                  "planned_bytes_by_row_blocks": p, "input_bytes": input_bytes(log_n), "device_free_bytes": free,
                  "device_total_bytes": total, "status": "not run: the smallest plan and the inputs exceed the free memory"})

    for log_n in args.profile_log_n:
        kernel_seconds(log_n, emit)


if __name__ == "__main__":
    main()
