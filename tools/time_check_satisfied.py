"""Time bj_check_satisfied and bj_lookup_multiplicities against one bj_prove on the same inputs, for the 2^22-row SHA-shaped
bench circuit (synthetic.generate(ctx, 22, 60, seed=42, lookup=True), fri_lde_factor 8, cap 16) and the 2^20-row
production-shaped circuit (synthetic.generate_production_shaped, fri_lde_factor 2, cap 32).  Each call is warmed up once, then
timed `repeats` times with a host clock around the call (both synchronise); the minimum and the median are reported.  Prints one
JSON line with the GPU name and power limit.  usage: time_check_satisfied.py [repeats=3]"""
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import era_boojum_b200 as bj  # noqa: E402
from era_boojum_b200 import prover, synthetic  # noqa: E402
from tools.prove_single_gpu_2p22 import gpu_power_limit_w  # noqa: E402


def timed(fn, repeats):
    fn()  # warm-up
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, {"min_s": round(min(ts), 4), "median_s": round(statistics.median(ts), 4)}


def measure(ctx, variables, sigmas, constants, gates, Q, lk, cfg, repeats):
    rep, check = timed(lambda: ctx.check_if_satisfied(variables, sigmas, constants, gates, lookup=lk), repeats)
    assert rep["satisfied"] == 1, rep
    mult, mult_t = timed(lambda: ctx.materialize_multiplicities_polynomials(variables, constants, lk), repeats)
    assert torch.equal(mult, lk["multiplicities"])
    nat = ctx.native_setup(sigmas, constants, gates, Q, cfg, lookup=lk)
    torch.cuda.synchronize()
    stages = {}
    t0 = time.perf_counter()
    nat.prove(variables, lk["multiplicities"], timings=stages)
    prove_s = time.perf_counter() - t0
    nat.close()
    ctx.synchronize()
    return {"rows_log2": variables.shape[1].bit_length() - 1, "variables": variables.shape[0], "check": check,
            "multiplicities": mult_t, "prove_s": round(prove_s, 3), "prove_quotient_stage_s": round(stages["3_quotient"], 3)}


def main():
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    ctx = bj.Context.on_current_stream(0)
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": gpu_power_limit_w(), "repeats": repeats}
    variables, sigmas, constants, gates, Q, lk = synthetic.generate(ctx, 22, 60, seed=42, lookup=True)
    cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)
    out["sha_2p22"] = measure(ctx, variables, sigmas, constants, gates, Q, lk, cfg, repeats)
    del variables, sigmas, constants, lk
    torch.cuda.empty_cache()
    c = synthetic.generate_production_shaped(ctx, 20, seed=0)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    out["production_2p20"] = measure(ctx, c["variables"], c["sigmas"], c["constants"], c["gates"], c["quotient_degree"],
                                     c["lookup"], cfg, repeats)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
