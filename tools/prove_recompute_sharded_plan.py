"""Prove the production-shaped circuit (synthetic.generate_production_shaped: 155 copy-permutation columns, 11 gates, 8 lookups
of width 3, quotient degree 8 over fri_lde_factor 2, cap 32) on N GPUs, one process per GPU over NCCL, under a per-rank
device-memory limit that forces the sharded recompute plan: every rank keeps no coset of the setup, witness and stage-2
columns, builds its trees one of its committed units at a time, evaluates its own quotient units one at a time, and rebuilds
the units the openings, DEEP and its query answers read (whole cosets at N <= 2, row blocks of n * 2 / N rows above it).

For every log_n given it prints (rank 0) one JSON line with each rank's plan, planned pool peak and pool high-water (setup +
first proof on a fresh context), the stage seconds of the fastest timed proof, the GPU name and power limit, whether every
rank returned the same proof, and `verified` from oracle/verifier.py.  With --check-single (default at 2^16) rank 0 also proves
the same inputs on one GPU on the resident plan and the sharded proof must equal it byte for byte.
usage:
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29513 \
      tools/prove_recompute_sharded_plan.py [--log-n 22 23] [--limit-gb G] [--rounds 3] [--hasher poseidon2|blake2s|keccak256]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import era_boojum_b200 as bj  # noqa: E402
from era_boojum_b200 import prover, synthetic  # noqa: E402
from oracle import verifier as OV  # noqa: E402


def gpu_power_limit_w(device):
    try:  # a read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(device)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def prove_single(c, cfg):
    """the single-GPU resident proof of the same inputs (JSON text)"""
    ctx = bj.Context.on_current_stream(torch.cuda.current_device())
    nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                           public_inputs=c["public_inputs"])
    proof = nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True)
    nat.close()
    ctx.synchronize()
    ctx.close()
    torch.cuda.empty_cache()
    return proof


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[22])
    ap.add_argument("--limit-gb", type=float, default=0, help="per-rank limit (default: the sharded recompute plan's bytes)")
    ap.add_argument("--check-single", type=int, nargs="*", default=[16], help="sizes also proved on one GPU and compared")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hasher", default="poseidon2")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda:%d" % local))
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100, hasher=args.hasher, transcript=args.hasher)
    gpu, power = torch.cuda.get_device_name(local), gpu_power_limit_w(local)
    for log_n in args.log_n:
        gen = bj.Context.on_current_stream(local)
        c = synthetic.generate_production_shaped(gen, log_n, seed=42)  # the same inputs on every rank
        torch.cuda.synchronize()
        gen.close()
        torch.cuda.empty_cache()
        lk = dict(width=c["lookup"]["width"], num_repetitions=c["lookup"]["num_repetitions"])
        shape = (log_n, c["sigmas"].shape[0], c["constants"].shape[0], c["quotient_degree"], cfg)
        plan = bj.proof_memory_plan(*shape, lookup=lk, world=world)
        plan["recompute_sharded"] = bj.proof_memory_plan_recompute_sharded(*shape, world, lookup=lk)
        limit = int(args.limit_gb * 1e9) if args.limit_gb else plan["recompute_sharded"]

        ctx = bj.Context.on_current_stream(local)
        comm = bj.Comm.from_torch_distributed(ctx, dist, cfg.fri_lde_factor)
        ctx.set_memory_limit(limit)
        ctx.allow_sharded_recompute_plan(True)
        ctx.memory_high_water(reset=True)
        t0 = time.perf_counter()
        nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], c["quotient_degree"], cfg, lookup=c["lookup"],
                               public_inputs=c["public_inputs"])
        torch.cuda.synchronize()
        setup_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        proof = nat.prove(c["variables"], c["lookup"]["multiplicities"], as_json=True)
        first_s = time.perf_counter() - t0
        high = ctx.memory_high_water()  # setup + first proof on a fresh context
        seconds, stages = [], []
        for _ in range(args.rounds):
            dist.barrier()
            tm = {}
            t0 = time.perf_counter()
            again = nat.prove(c["variables"], c["lookup"]["multiplicities"], timings=tm, as_json=True)
            seconds.append(round(time.perf_counter() - t0, 4))
            stages.append(tm)
            assert again == proof, "a proof of the same inputs moved"
        mp = nat.memory_plan()
        best = min(range(len(stages)), key=lambda i: sum(stages[i].values())) if stages else None
        mine = {"rank": rank, "plan": nat.plan, "chunk": mp["chunk"], "planned_pool_peak_bytes": mp["pool"],
                "planned_outside_pool_bytes": mp["outside_pool"], "pool_high_water_bytes": high,
                "high_water_equals_plan": high == mp["pool"], "setup_seconds": round(setup_s, 3),
                "first_prove_seconds": round(first_s, 3), "prove_seconds": seconds,
                "stage_seconds": {k: round(v, 4) for k, v in stages[best].items()} if stages else {},
                "proof_sha256": hashlib.sha256(proof.encode()).hexdigest()}
        vk = nat.vk()
        nat.close()
        ctx.synchronize()
        comm.close()
        ctx.close()
        torch.cuda.empty_cache()
        ranks = [None] * world
        dist.all_gather_object(ranks, mine)
        if rank == 0:
            out = {"workload": "production-shaped circuit 2^%d x 155 columns, 11 gates, Q = 8 over L = 2, cap 32, %s" % (log_n, args.hasher),
                   "world": world, "row_blocks_per_coset": max(1, world // 2), "gpu": gpu, "power_limit_w": power,
                   "planned_bytes": plan, "limit_bytes": limit,
                   "same_proof_on_every_rank": len({r["proof_sha256"] for r in ranks}) == 1, "ranks": ranks}
            if log_n in args.check_single:
                out["identical_to_single_gpu_resident"] = prove_single(c, cfg) == proof
            t0 = time.perf_counter()
            out["verified"] = bool(OV.verify(vk, json.loads(proof)))
            out["verify_cpu_seconds"] = round(time.perf_counter() - t0, 2)
            print(json.dumps(out), flush=True)
            assert out["verified"] and out["same_proof_on_every_rank"] and out.get("identical_to_single_gpu_resident", True)
        del c
        torch.cuda.empty_cache()
        dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
