"""Prove the production-shaped circuit (synthetic.generate_production_shaped: the geometry of the reference's vk.json - 155
copy-permutation columns, 11 gates, 8 lookups of width 3, quotient degree 8 over fri_lde_factor 2, cap 32) on ONE GPU under a
device-memory limit that forces the streamed plan: the setup, witness and stage-2 columns are kept on cosets [0, 2) only and
the quotient evaluates them onto cosets [2, 8) one at a time.

For every log_n given (default 20 and 22) it prints one JSON line with the chosen plan, planned pool peak, pool high-water
(setup + first proof on a fresh context), stage seconds, the GPU name and power limit and `verified` from oracle/verifier.py.
With --compare (default at 2^20) the resident plan proves the same inputs on a second context and the two are timed in
alternating rounds; the proofs must be byte-identical.
usage: prove_production_shape_limited.py [--log-n 20 22] [--compare 20] [--rounds 3] [--hasher poseidon2|blake2s]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import era_boojum_b200 as bj  # noqa: E402
from era_boojum_b200 import prover, synthetic  # noqa: E402
from oracle import verifier as OV  # noqa: E402


def gpu_power_limit_w():
    try:  # a read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


class Run:
    """one context, one setup under `limit` (0: what the device has free) and its proofs"""

    def __init__(self, c, cfg, limit):
        self.c = c
        self.ctx = bj.Context.on_current_stream(0)
        self.ctx.set_memory_limit(limit)
        self.ctx.memory_high_water(reset=True)
        t0 = time.perf_counter()
        self.nat = self.ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                                         public_inputs=c["public_inputs"])
        torch.cuda.synchronize()
        self.setup_s = time.perf_counter() - t0
        self.plan = self.nat.plan
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
        return {"plan": self.plan, "planned_pool_peak_bytes": mp["pool"], "planned_outside_pool_bytes": mp["outside_pool"],
                "pool_high_water_bytes": self.high_water, "setup_seconds": round(self.setup_s, 3),
                "first_prove_seconds": round(self.first_s, 3), "prove_seconds": self.seconds,
                "stage_seconds": {k: round(v, 4) for k, v in self.stages[best].items()}}

    def close(self):
        self.nat.close()
        self.ctx.synchronize()
        self.ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--compare", type=int, nargs="*", default=[20], help="sizes also proved on the resident plan, alternated")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hasher", default="poseidon2")
    args = ap.parse_args()
    gpu, power = torch.cuda.get_device_name(0), gpu_power_limit_w()
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100, hasher=args.hasher, transcript=args.hasher)
    for log_n in args.log_n:
        gen = bj.Context.on_current_stream(0)
        c = synthetic.generate_production_shaped(gen, log_n, seed=42)
        torch.cuda.synchronize()
        gen.close()
        torch.cuda.empty_cache()  # the generator's temporaries go back to the device for the prover's pool
        lk = dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"])
        plan = bj.proof_memory_plan(log_n, c["sigmas"].shape[0], c["constants"].shape[0], c["quotient_degree"], cfg, lookup=lk)
        out = {"workload": "production-shaped circuit 2^%d x 155 columns, 11 gates, Q = 8 over L = 2, cap 32, %s" % (log_n, args.hasher),
               "gpu": gpu, "power_limit_w": power, "planned_bytes": plan, "limit_bytes": plan["streamed"]}
        streamed = Run(c, cfg, plan["streamed"])
        assert streamed.plan == "streamed", streamed.plan
        resident = Run(c, cfg, 0) if log_n in args.compare else None
        if resident:
            assert resident.plan == "resident", resident.plan
            out["identical_to_resident"] = resident.proof == streamed.proof
        for _ in range(args.rounds):  # alternating, so that both plans see the same state of a shared device
            streamed.timed()
            if resident:
                resident.timed()
        out["streamed"] = streamed.report()
        if resident:
            out["resident"] = resident.report()
            resident.close()
        t0 = time.perf_counter()
        out["verified"] = bool(OV.verify(streamed.nat.vk(), json.loads(streamed.proof)))
        out["verify_cpu_seconds"] = round(time.perf_counter() - t0, 2)
        streamed.close()
        del c
        torch.cuda.empty_cache()
        print(json.dumps(out), flush=True)
        assert out["verified"] and out.get("identical_to_resident", True)


if __name__ == "__main__":
    main()
