"""torchrun: per-rank stage timings of the coset-sharded prover (both hasher configurations).
--production-shape: the native driver (bj_prove over NCCL) on the production-shaped circuit (155 columns, quotient degree 8
over LDE factor 2, cap 32); with more ranks than the 2 cosets every coset is split into world / 2 row blocks (up to 16 ranks).
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N tools/prove_sharded_time.py [--production-shape]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.distributed as dist
import era_boojum_b200 as bj
from era_boojum_b200 import parallel, prover, synthetic
rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda:%d" % local))
world = dist.get_world_size()
log_n = int(os.environ.get("LOG_N", "22"))
if "--production-shape" in sys.argv[1:]:
    log_n = int(os.environ.get("LOG_N", "20"))
    ctx = bj.Context.on_current_stream(local)
    comm = bj.Comm.from_torch_distributed(ctx, dist, 2)
    c = synthetic.generate_production_shaped(ctx, log_n, seed=5)
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    nat = ctx.native_setup(c["sigmas"], c["constants"], c["gates"], 8, cfg, lookup=c["lookup"], public_inputs=c["public_inputs"])
    nat.prove(c["variables"], c["lookup"]["multiplicities"])
    for _ in range(2):
        torch.cuda.synchronize(); dist.barrier()
        tm = {}
        t0 = time.perf_counter()
        nat.prove(c["variables"], c["lookup"]["multiplicities"], timings=tm)
        torch.cuda.synchronize()
        print("rank", rank, "world", world, "production-shape log_n", log_n, round(time.perf_counter() - t0, 4),
              {k: round(v, 4) for k, v in tm.items()}, flush=True)
    nat.close()
    comm.close()
    dist.destroy_process_group()
    sys.exit(0)
ctx = bj.Context.on_current_stream(local)
ctx.set_coset_shard(rank, world, 8)
comm = parallel.TorchDistComm(dist)
variables, sigmas, constants, gates, Q, lk = synthetic.generate(ctx, log_n, 60, seed=42, lookup=True)
for hasher in ("poseidon2", "blake2s", "blake2s"):
    cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100, hasher=hasher, transcript=hasher)
    setup = prover.Setup(ctx, sigmas, constants, gates, Q, cfg, lookup=lk, comm=comm)
    prover.prove(ctx, setup, variables, multiplicities=lk["multiplicities"])
    torch.cuda.synchronize(); dist.barrier()
    tm = {}
    t0 = time.perf_counter()
    prover.prove(ctx, setup, variables, timings=tm, multiplicities=lk["multiplicities"])
    torch.cuda.synchronize()
    print("rank", rank, hasher, round(time.perf_counter() - t0, 4), {k: round(v, 4) for k, v in tm.items()}, flush=True)
    del setup
    torch.cuda.empty_cache()
    dist.barrier()
dist.destroy_process_group()
