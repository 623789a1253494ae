"""torchrun check on N GPUs: column-sharded iNTT -> NCCL all-gather of monomials -> coset-sharded LDE + Merkle subtrees
-> all-gather of caps equals the single-GPU commitment (bit-exact), plus timings; then the coset-sharded prover
(prover.prove with a TorchDistComm) must return the single-GPU proof on every rank, and so must the library's driver
(bj_prove over NCCL) on the SHA-bench shape and on the production shape (LDE factor 2: cosets split into row blocks above
2 ranks).  The first parts use LDE factor 8 and so need N <= 8.  Usage:
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 tools/multi_gpu_check.py"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist
import era_boojum_b200 as bj
from era_boojum_b200 import parallel

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda:%d" % local))
ctx = bj.Context.on_current_stream(local)
log_n = int(os.environ.get("LOG_N", "20"))
V, L, cap = 64, 8, 16
gen = torch.Generator(device="cuda:%d" % local)
gen.manual_seed(123)   # same data on every rank
cols = torch.randint(0, 2**63 - 1, (V, 1 << log_n), dtype=torch.int64, device="cuda:%d" % local, generator=gen)
blk = parallel.column_block(rank, world, V)
backend = parallel.TorchBackend(ctx)
res = parallel.commit_sharded(backend, dist, cols[blk.start:blk.stop].contiguous(), V, L, cap)
torch.cuda.synchronize(); dist.barrier()
t0 = time.perf_counter()
for _ in range(3):
    res = parallel.commit_sharded(backend, dist, cols[blk.start:blk.stop].contiguous(), V, L, cap)
torch.cuda.synchronize(); dist.barrier()
t_sharded = (time.perf_counter() - t0) / 3
# single-GPU reference commitment, computed redundantly on every rank
lde = ctx.transform_raw_storages_to_lde(cols, L)
tree = ctx.merkle_tree_construct([lde[c].reshape(-1) for c in range(V)], cap)
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(3):
    lde = ctx.transform_raw_storages_to_lde(cols, L)
    tree = ctx.merkle_tree_construct([lde[c].reshape(-1) for c in range(V)], cap)
torch.cuda.synchronize()
t_single = (time.perf_counter() - t0) / 3
ok = np.array_equal(bj.to_numpy(res["cap"]), tree.get_cap())
for j, ev in res["cosets"].items():
    ok = ok and bool(torch.equal(ev, lde[:, j, :]))
flag = torch.tensor([1 if ok else 0], device="cuda:%d" % local)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print({"world": world, "log_n": log_n, "cols": V, "bit_identical_to_single_gpu": bool(flag.item()),
           "commit_sharded_s": round(t_sharded, 4), "commit_single_gpu_s": round(t_single, 4),
           "speedup": round(t_single / t_sharded, 2)})
del lde, tree, res, cols
torch.cuda.empty_cache()

# ---- coset-sharded PROVER over NCCL == single-GPU prover (same proof, bit for bit), and the oracle verifier accepts ----
import json
from era_boojum_b200 import prover, synthetic
p_log_n = int(os.environ.get("PROVE_LOG_N", "16"))
cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100)
variables, sigmas, constants, gates, Q, lk = synthetic.generate(ctx, p_log_n, 60, seed=7, lookup=True)
single = prover.prove(ctx, prover.Setup(ctx, sigmas, constants, gates, Q, cfg, lookup=lk), variables, multiplicities=lk["multiplicities"])
sctx = bj.Context.on_current_stream(local)
sctx.set_coset_shard(rank, world, 8)
setup = prover.Setup(sctx, sigmas, constants, gates, Q, cfg, lookup=lk, comm=parallel.TorchDistComm(dist))
sharded = prover.prove(sctx, setup, variables, multiplicities=lk["multiplicities"])
same = json.dumps(single, sort_keys=True) == json.dumps(sharded, sort_keys=True)
flag = torch.tensor([1 if same else 0], device="cuda:%d" % local)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    from oracle import verifier as OV
    print({"world": world, "prove_log_n": p_log_n, "sharded_proof_equals_single_gpu_proof_on_every_rank": bool(flag.item()),
           "oracle_verifier_accepts": bool(OV.verify(setup.vk(), sharded))})
del setup, sctx
torch.cuda.empty_cache()

# ---- the library's own sharded driver: bj_prove on contexts that carry a bj_comm over NCCL (csrc/comm.cu) ----
nctx = bj.Context.on_current_stream(local)
comm = bj.Comm.from_torch_distributed(nctx, dist, 8)
for hasher, transcript in (("poseidon2", "poseidon"), ("blake2s", "blake2s")):
    cfg = prover.ProofConfig(fri_lde_factor=8, merkle_tree_cap_size=16, security_level=100, hasher=hasher, transcript=transcript)
    ref = ctx.native_setup(sigmas, constants, gates, Q, cfg, lookup=lk)
    want = ref.prove(variables, lk["multiplicities"])
    ref_cap = ref.get_cap()
    ref.close()
    nat = nctx.native_setup(sigmas, constants, gates, Q, cfg, lookup=lk)
    nat.prove(variables, lk["multiplicities"])
    torch.cuda.synchronize(); dist.barrier()
    tm = {}
    t0 = time.perf_counter()
    got = nat.prove(variables, lk["multiplicities"], timings=tm)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    same = json.dumps(want, sort_keys=True) == json.dumps(got, sort_keys=True) and np.array_equal(ref_cap, nat.get_cap())
    flag = torch.tensor([1 if same else 0], device="cuda:%d" % local)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print({"world": world, "native_nccl_sharded_bj_prove": hasher + "+" + transcript, "equals_single_gpu_proof_on_every_rank": bool(flag.item()),
               "oracle_verifier_accepts": bool(OV.verify(nat.vk(), got)), "seconds": round(dt, 4),
               "stages_s": {k: round(v, 4) for k, v in tm.items()}})
    nat.close()
comm.close()

# ---- the production shape (LDE factor 2, quotient degree 8, cap 32) through bj_prove over NCCL: with more ranks than its
#      2 cosets every coset is split into world / 2 row blocks (up to 16 ranks) ----
prod_log_n = int(os.environ.get("PROD_LOG_N", "14"))
pctx = bj.Context.on_current_stream(local)
pcomm = bj.Comm.from_torch_distributed(pctx, dist, 2)
pc = synthetic.generate_production_shaped(ctx, prod_log_n, seed=5)
pcfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
m = pc["lookup"]["multiplicities"]
ref = ctx.native_setup(pc["sigmas"], pc["constants"], pc["gates"], 8, pcfg, lookup=pc["lookup"], public_inputs=pc["public_inputs"])
want = ref.prove(pc["variables"], m)
ref_cap = ref.get_cap()
ref.close()
nat = pctx.native_setup(pc["sigmas"], pc["constants"], pc["gates"], 8, pcfg, lookup=pc["lookup"], public_inputs=pc["public_inputs"])
got = nat.prove(pc["variables"], m)
same = json.dumps(want, sort_keys=True) == json.dumps(got, sort_keys=True) and np.array_equal(ref_cap, nat.get_cap())
flag = torch.tensor([1 if same else 0], device="cuda:%d" % local)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print({"world": world, "production_shaped_log_n": prod_log_n, "row_blocks_per_coset": max(1, world // 2),
           "equals_single_gpu_proof_on_every_rank": bool(flag.item()), "oracle_verifier_accepts": bool(OV.verify(nat.vk(), got))})
nat.close()
pcomm.close()
dist.destroy_process_group()
