"""Prove the 2^22-row SHA-shaped bench circuit (synthetic.generate: 60 general-purpose + 32 lookup columns, 8 lookups of width 4,
quotient degree 4, fri_lde_factor 8, cap 16) on ONE GPU.  The resident memory plan does not fit an 80 GB H100 at this size, so
bj_setup_create picks the compact plan under the default limit (what the device has free): cosets [4, 8) of the setup, witness
and stage-2 columns are recomputed for DEEP and the query answers instead of being kept.  Proves once per hasher / transcript
pair of bench.py, checks every proof with the oracle verifier and prints one JSON line: stage seconds, plan bytes, pool
high-water, GPU name and power limit.  usage: prove_single_gpu_2p22.py [log_n=22]"""
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

STAGES = ("1_witness_lde_commit", "2_stage2_products_lde_commit", "3_quotient", "4_openings", "5_deep_fri", "6_queries")


def gpu_power_limit_w():
    try:  # a read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    log_n = int(sys.argv[1]) if len(sys.argv) > 1 else 22
    ctx = bj.Context.on_current_stream(0)
    variables, sigmas, constants, gates, Q, lk = synthetic.generate(ctx, log_n, 60, seed=42, lookup=True)
    torch.cuda.synchronize()
    out = {"rows_log2": log_n, "gpu": torch.cuda.get_device_name(0), "power_limit_w": gpu_power_limit_w(), "proofs": {}}
    for hasher, transcript in (("poseidon2", "poseidon"), ("blake2s", "blake2s")):
        cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100, hasher=hasher, transcript=transcript)
        plan = bj.proof_memory_plan(log_n, variables.shape[0], constants.shape[0], Q, cfg, lookup=lk)
        ctx.memory_high_water(reset=True)
        name = "%s/%s" % (hasher, transcript)
        try:
            t0 = time.perf_counter()
            nat = ctx.native_setup(sigmas, constants, gates, Q, cfg, lookup=lk)
            torch.cuda.synchronize()
            setup_s = time.perf_counter() - t0
            timings = {}
            t0 = time.perf_counter()
            proof = nat.prove(variables, lk["multiplicities"], timings=timings)
            prove_s = time.perf_counter() - t0
        except bj.BoojumError as e:
            out["proofs"][name] = {"error": str(e), "plan_bytes": plan, "pool_high_water_bytes": ctx.memory_high_water()}
            print(json.dumps(out))
            raise
        high = ctx.memory_high_water()
        ok = OV.verify(nat.vk(), proof)
        out["proofs"][name] = {
            "plan": "compact" if nat.compact else "resident", "plan_bytes": plan, "pool_high_water_bytes": high,
            "setup_seconds": round(setup_s, 3), "prove_seconds": round(prove_s, 3),
            "stage_seconds": {k: round(timings[k], 3) for k in STAGES}, "verified": bool(ok)}
        nat.close()
        ctx.synchronize()
        assert ok, "the oracle verifier rejected the %s/%s proof" % (hasher, transcript)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
