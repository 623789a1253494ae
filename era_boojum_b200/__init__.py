"""era_boojum_b200 - H100-native backend for Boojum's polynomial-commitment hot path.

Python host mirror of the reference plug points, over the C-ABI (libboojum_b200.so):

    reference (Rust, era-boojum src/)                        here
    --------------------------------------------------------     -------------------------------------------
    Worker (worker/mod.rs:5-87)                                   Context (device + stream + cached tables)
    P::fft_natural_to_bitreversed (field/traits/field_like.rs)    Context.fft_natural_to_bitreversed
    P::ifft_natural_to_natural                                    Context.ifft_natural_to_natural
    precompute_twiddles_for_fft (cs/implementations/utils.rs)     Context.precompute_twiddles_for_fft
    transform_raw_storages_to_lde (utils.rs:270-309)              Context.transform_raw_storages_to_lde
    MerkleTreeWithCap::construct* (cs/oracle/merkle_tree.rs)      Context.merkle_tree_construct -> MerkleTreeWithCap
    fold step of do_fri (cs/implementations/fri/mod.rs)           Context.fri_fold

Tensors are torch int64 CUDA tensors holding the u64 bit patterns (torch is plumbing: memory + streams).
No CPU fallback exists: importing this package without the built library raises, and creating a Context
without a CUDA device raises BoojumError(BJ_ERR_NO_DEVICE).
"""
import ctypes
import itertools

import numpy as np

from . import native
from .native import BoojumError, P, lib

__all__ = ["Context", "Comm", "compile_gate_programs", "MerkleTreeWithCap", "Transcript", "FriOracles", "BoojumError", "P", "to_device", "to_numpy"]


class Transcript:
    """GoldilocksPoisedon2Transcript (cs/implementations/transcript.rs:62-129, 140-151) - host side."""

    def __init__(self, kind="poseidon2"):
        """kind: "poseidon2" (GoldilocksPoisedon2Transcript), "blake2s" (Blake2sTranscript, transcript.rs:155-260), "keccak256"
        (Keccak256Transcript, :262-367) or "poseidon" (GoldilocksPoisedonTranscript, :131-138, the sponge transcript over the
        Poseidon v1 permutation: the TR of the reference's recursive-mode SHA-256 benches)."""
        self.kind = kind
        new = {"poseidon2": lib.bj_transcript_new, "blake2s": lib.bj_transcript_new_blake2s, "keccak256": lib.bj_transcript_new_keccak256,
               "poseidon": lib.bj_transcript_new_poseidon}
        self._h = ctypes.c_void_p(new[kind]())

    def witness_field_elements(self, els):
        a = np.ascontiguousarray(np.array([int(e) for e in els], dtype=np.uint64))
        lib.bj_transcript_witness_field_elements(self._h, a.ctypes.data_as(ctypes.c_void_p), a.shape[0])

    def witness_merkle_tree_cap(self, cap):
        a = np.ascontiguousarray(np.array(cap, dtype=np.uint64).reshape(-1, 4))
        lib.bj_transcript_witness_merkle_tree_cap(self._h, a.ctypes.data_as(ctypes.c_void_p), a.shape[0])

    def get_challenge(self):
        return int(lib.bj_transcript_get_challenge(self._h))

    def get_multiple_challenges_fixed(self, n=2):
        return tuple(self.get_challenge() for _ in range(n))

    def get_index_bits(self, num_bits, max_needed):
        """BoolsBuffer::get_bits (transcript.rs:369-417) packed LSB first."""
        return int(lib.bj_transcript_get_index_bits(self._h, num_bits, max_needed))

    def __del__(self):
        if getattr(self, "_h", None):
            lib.bj_transcript_free(self._h)
            self._h = None


def _ok(status, what="libboojum_b200 call"):
    """status check for context-free C-ABI calls (never inside an `assert`: `python -O` would drop the call itself)."""
    if status != 0:
        raise BoojumError(status, "%s: %s" % (what, lib.bj_status_string(status).decode()))


def _shard_split(world, lde_degree):
    """log2 of the row blocks per coset of a domain shard of `world` ranks (0: every rank holds whole cosets)"""
    return max(0, world.bit_length() - lde_degree.bit_length())


class FriOracles:
    """FriOracles (cs/implementations/fri/mod.rs:36-47): base + intermediate oracle caps, monomial forms, queries."""

    def __init__(self, handle, cap_size, keepalive):
        self._h, self.cap_size, self._keep = handle, cap_size, keepalive

    def num_oracles(self):
        return int(lib.bj_fri_oracles_num_oracles(self._h))

    def get_cap(self, i):
        out = np.zeros((self.cap_size, 4), np.uint64)
        _ok(lib.bj_fri_oracles_get_cap(self._h, i, out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def monomial_forms(self):
        n = int(lib.bj_fri_oracles_num_monomials(self._h))
        c0, c1 = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        _ok(lib.bj_fri_oracles_get_monomials(self._h, c0.ctypes.data_as(ctypes.c_void_p), c1.ctypes.data_as(ctypes.c_void_p)))
        return c0, c1

    def challenges(self):
        out = np.zeros((self.num_oracles(), 2), np.uint64)
        _ok(lib.bj_fri_oracles_get_challenges(self._h, out.ctypes.data_as(ctypes.c_void_p)))
        return [tuple(int(x) for x in r) for r in out]

    def query(self, oracle_idx, leaf_index, log_fold):
        le = np.zeros(2 << log_fold, np.uint64)
        path = np.zeros((40, 4), np.uint64)
        plen = ctypes.c_uint32()
        st = lib.bj_fri_oracles_query(self._h, oracle_idx, leaf_index, le.ctypes.data_as(ctypes.c_void_p),
                                      path.ctypes.data_as(ctypes.c_void_p), ctypes.byref(plen))
        if st != 0:
            raise BoojumError(st, "bj_fri_oracles_query")
        return le, path[: plen.value]

    def close(self):
        if getattr(self, "_h", None):
            lib.bj_fri_oracles_free(self._h)
            self._h = None

    def __del__(self):
        self.close()


def compile_gate_programs(gates, n_variables, n_witnesses, n_constants, peephole=15):
    """bj_gate_programs_compile: what the gate evaluator will execute for these gate dicts - host code only (no GPU needed).
    Returns (records [n, 4] uint64 in the step format documented in include/boojum_b200.h, first record of every gate + the
    end, maximal number of live temporaries)."""
    keep, descs = Context._gate_descs(gates)
    n = ctypes.c_uint64()
    live = ctypes.c_uint32()
    first = (ctypes.c_uint32 * (len(gates) + 1))()
    _ok(lib.bj_gate_programs_compile(descs, len(gates), n_variables, n_witnesses, n_constants, peephole, None, 0, ctypes.byref(n),
                                     first, ctypes.byref(live)), "bj_gate_programs_compile")
    rec = np.zeros((max(1, n.value), 4), np.uint64)
    _ok(lib.bj_gate_programs_compile(descs, len(gates), n_variables, n_witnesses, n_constants, peephole,
                                     rec.ctypes.data_as(ctypes.c_void_p), rec.shape[0], ctypes.byref(n), first, ctypes.byref(live)),
        "bj_gate_programs_compile")
    del keep
    return rec[: n.value], list(first), int(live.value)


def to_device(a, device="cuda:0"):
    """numpy uint64 array -> torch int64 CUDA tensor (same bits)."""
    import torch
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return torch.from_numpy(a.view(np.int64)).to(device)


def to_numpy(t):
    """torch int64 tensor -> numpy uint64 array (same bits)."""
    return t.detach().cpu().numpy().view(np.uint64)


class MerkleTreeWithCap:
    """cap_size / leaf_hashes / node_hashes_enumerated_from_leafs (cs/oracle/merkle_tree.rs:23-33)."""

    def __init__(self, cap_size, leaf_hashes, nodes):
        self.cap_size = cap_size
        self.leaf_hashes = leaf_hashes  # [n_leaves, 4] int64 cuda
        self.nodes = nodes              # [n_leaves - cap_size, 4]

    def levels(self):
        out, off, cnt = [], 0, self.leaf_hashes.shape[0]
        while cnt > self.cap_size:
            cnt //= 2
            out.append(self.nodes[off:off + cnt])
            off += cnt
        return out

    def get_cap(self):
        """get_cap (merkle_tree.rs:451-460): canonical digests of the level with cap_size nodes."""
        lv = self.levels()
        return to_numpy(lv[-1] if lv else self.leaf_hashes)

    def get_proof(self, idx):
        """get_proof (merkle_tree.rs:462-480): (leaf hash, siblings bottom-up, cap level excluded)."""
        lv = self.levels()
        layers = ([self.leaf_hashes] + lv[:-1]) if lv else []
        leaf = to_numpy(self.leaf_hashes[idx])
        path = []
        for layer in layers:
            path.append(to_numpy(layer[idx ^ 1]))
            idx >>= 1
        return leaf, np.array(path, dtype=np.uint64).reshape(-1, 4)


class Context:
    """One device + one stream (the reference's Worker role)."""

    def __init__(self, device=0, stream=None):
        import torch
        self._torch = torch
        self.device = device
        handle = ctypes.c_void_p()
        st = lib.bj_ctx_create(device, ctypes.c_void_p(stream) if stream else None, ctypes.byref(handle))
        if st != native.BJ_OK:
            raise BoojumError(st, lib.bj_status_string(st).decode())
        self._h = handle
        self._stream = stream
        import weakref
        self._children = weakref.WeakSet()   # library objects that hold device memory of this context (freed before it)

    @classmethod
    def on_current_stream(cls, device=0):
        import torch
        with torch.cuda.device(device):
            return cls(device, torch.cuda.current_stream().cuda_stream)

    def close(self):
        if self._h:
            for child in list(self._children):
                child.close()
            lib.bj_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st):
        if st != native.BJ_OK:
            raise BoojumError(st, "%s: %s" % (lib.bj_status_string(st).decode(), lib.bj_last_error(self._h).decode()))

    def synchronize(self):
        self._check(lib.bj_ctx_synchronize(self._h))

    def lane(self):
        """bj_ctx_create_lane: a context on this one's device with its own stream and pool that proves against this
        context's setups (NativeSetup.prove(..., ctx=lane)), concurrently with the other lanes from other threads.  It
        inherits the memory limit and the recompute-plan switch; closing this context closes its lanes first."""
        h = ctypes.c_void_p()
        self._check(lib.bj_ctx_create_lane(self._h, ctypes.byref(h)))
        import weakref
        lane = Context.__new__(Context)
        lane._torch, lane.device, lane._h, lane._stream = self._torch, self.device, h, None
        lane._children = weakref.WeakSet()
        lane.parent = self
        self._children.add(lane)
        return lane

    shard_rank, shard_world, shard_split = 0, 1, 0

    def set_coset_shard(self, rank, world, lde_degree):
        """bj_ctx_set_coset_shard: this context holds the LDE cosets j = rank (mod world) of every committed polynomial
        (multi-GPU proving, one process per GPU).  Sizes passed to the C-ABI stay global; tensors are local."""
        self._check(lib.bj_ctx_set_coset_shard(self._h, rank, world, lde_degree.bit_length() - 1))
        self.shard_rank, self.shard_world, self.shard_split = rank, world, 0

    def set_domain_shard(self, rank, world, lde_degree):
        """bj_ctx_set_domain_shard: set_coset_shard for world <= lde_degree; above it every coset is cut into
        B = world / lde_degree row blocks (units) and this context holds the units u = rank (mod world), [local unit][n / B]."""
        self._check(lib.bj_ctx_set_domain_shard(self._h, rank, world, lde_degree.bit_length() - 1))
        self.shard_rank, self.shard_world = rank, world
        self.shard_split = _shard_split(world, lde_degree)

    def launch_count(self):
        return int(lib.bj_launch_count(self._h))

    def set_memory_limit(self, nbytes):
        """bj_ctx_set_memory_limit: device bytes a proof on this context may use (0: what is free when the setup is created).
        native_setup picks the resident plan if it fits, else the compact one (quotient degree < LDE factor, one GPU), else the
        streamed one (quotient degree > LDE factor, one GPU or a sharded context), and raises BoojumError (out of device
        memory, with every applicable plan's byte count) if none does."""
        self._check(lib.bj_ctx_set_memory_limit(self._h, int(nbytes)))

    def allow_recompute_plan(self, allow=True):
        """bj_ctx_allow_recompute_plan: with allow, native_setup falls back to the recompute plan (one GPU, any quotient degree;
        no coset of the setup, witness or stage-2 columns kept, every reader rebuilds the cosets it needs, so slower) when no
        other plan fits under the limit.  Off by default; a sharded context ignores it."""
        self._check(lib.bj_ctx_allow_recompute_plan(self._h, int(bool(allow))))

    def set_max_row_blocks(self, max_blocks):
        """bj_ctx_set_max_row_blocks: row blocks per coset (1, the default, 2, 4 or 8) the one-GPU recompute plan may cut its
        trees and quotient into.  When native_setup takes the recompute plan it takes the fewest row blocks whose plan
        (proof_memory_plan_recompute_blocks) fits; NativeSetup.row_blocks reports them.  A context with a communicator ignores
        it; lanes inherit it."""
        self._check(lib.bj_ctx_set_max_row_blocks(self._h, int(max_blocks)))

    def allow_sharded_recompute_plan(self, allow=True):
        """bj_ctx_allow_sharded_recompute_plan: with allow, native_setup on a context with a communicator falls back to the
        recompute plan on this rank (proof_memory_plan_recompute_sharded) when neither the resident nor the streamed plan fits
        under the rank's limit.  Off by default; a context without a communicator ignores it."""
        self._check(lib.bj_ctx_allow_sharded_recompute_plan(self._h, int(bool(allow))))

    def memory_high_water(self, reset=False):
        """bj_ctx_memory_high_water: the highest device memory the context's pool has had in use (bytes)"""
        v = ctypes.c_uint64()
        self._check(lib.bj_ctx_memory_high_water(self._h, ctypes.byref(v), int(bool(reset))))
        return int(v.value)

    @staticmethod
    def _ptr(t):
        return ctypes.c_void_p(t.data_ptr())

    def _cols(self, t):
        assert t.is_cuda and t.dtype == self._torch.int64 and t.is_contiguous()
        n = t.shape[-1]
        assert n & (n - 1) == 0
        return n.bit_length() - 1, t.numel() // n, n

    # ---- NTT family ----
    def precompute_twiddles_for_fft(self, fft_size, inverse=False):
        log_n = fft_size.bit_length() - 1
        out = self._torch.empty(max(1, fft_size // 2), dtype=self._torch.int64, device="cuda:%d" % self.device)
        self._check(lib.bj_twiddles(self._h, log_n, int(inverse), self._ptr(out)))
        return out

    def fft_natural_to_bitreversed(self, cols, coset=1):
        """In place on a [n_cols, n] (or [n]) tensor."""
        log_n, n_cols, n = self._cols(cols)
        self._check(lib.bj_ntt_natural_to_bitreversed(self._h, self._ptr(cols), log_n, n_cols, n, coset))
        return cols

    def ifft_natural_to_natural(self, cols, coset=1):
        log_n, n_cols, n = self._cols(cols)
        self._check(lib.bj_intt_natural_to_natural(self._h, self._ptr(cols), log_n, n_cols, n, coset))
        return cols

    def bitreverse_enumeration_inplace(self, cols):
        log_n, n_cols, n = self._cols(cols)
        self._check(lib.bj_bitreverse(self._h, self._ptr(cols), log_n, n_cols, n))
        return cols

    def transform_raw_storages_to_lde(self, cols, lde_degree, from_monomials=False, out=None, next_row=False):
        """[n_cols, n] Lagrange values -> [n_cols, lde_degree, n] (coset-major, bit-reversed in coset).  A shard produces
        only its own units: [n_cols, (lde_degree * B) // world, n // B] with B row blocks per coset (B = 1: whole cosets).
        next_row: the LDE of f(w_n x) instead (bj_lde_next_row)."""
        log_n, n_cols, n = self._cols(cols)
        log_l = lde_degree.bit_length() - 1
        if out is None:
            b = 1 << self.shard_split
            out = self._torch.empty((n_cols, max(1, lde_degree * b // self.shard_world), n // b), dtype=self._torch.int64,
                                    device=cols.device)
        fn = lib.bj_lde_next_row if next_row else lib.bj_lde
        self._check(fn(self._h, self._ptr(cols), n, self._ptr(out), log_n, log_l, n_cols, int(from_monomials)))
        return out

    # ---- Merkle ----
    def merkle_tree_construct(self, sources, cap_size, elems_per_leaf=1, hasher="poseidon2"):
        """sources: list of flat int64 CUDA tensors in leaf-preimage order (MerkleTreeWithCap::construct for
        elems_per_leaf == 1, construct_by_chunking[_from_flat_sources] otherwise)."""
        torch = self._torch
        n_leaves = sources[0].numel() // elems_per_leaf
        for s in sources:
            assert s.is_cuda and s.dtype == torch.int64 and s.is_contiguous() and s.numel() == n_leaves * elems_per_leaf
        ptrs = (ctypes.c_void_p * len(sources))(*[s.data_ptr() for s in sources])
        dev = sources[0].device
        leaf_hashes = torch.empty((n_leaves, 4), dtype=torch.int64, device=dev)
        nodes = torch.empty((max(n_leaves - cap_size, 1), 4), dtype=torch.int64, device=dev)
        build = {"poseidon2": lib.bj_merkle_build_poseidon2, "blake2s": lib.bj_merkle_build_blake2s,
                 "keccak256": lib.bj_merkle_build_keccak256}[hasher]
        self._check(build(self._h, ptrs, len(sources), n_leaves, elems_per_leaf, cap_size, self._ptr(leaf_hashes), self._ptr(nodes)))
        return MerkleTreeWithCap(cap_size, leaf_hashes, nodes[:max(n_leaves - cap_size, 0)])

    def poseidon2_hash_rows(self, rows):
        torch = self._torch
        assert rows.is_cuda and rows.dtype == torch.int64 and rows.is_contiguous() and rows.dim() == 2
        out = torch.empty((rows.shape[0], 4), dtype=torch.int64, device=rows.device)
        self._check(lib.bj_poseidon2_hash_rows(self._h, self._ptr(rows), rows.shape[0], rows.shape[1], self._ptr(out)))
        return out

    def poseidon2_permute(self, states):
        assert states.is_cuda and states.is_contiguous() and states.shape[-1] == 12
        self._check(lib.bj_poseidon2_permute(self._h, self._ptr(states), states.numel() // 12))
        return states

    # ---- element-wise ----
    def batch_inverse_inplace(self, a):
        """batch_inverse_inplace (cs/implementations/utils.rs:439-472); zero -> zero."""
        self._check(lib.bj_batch_inverse(self._h, self._ptr(a), a.numel()))
        return a

    def batch_inverse_inplace_in_extension(self, c0, c1):
        self._check(lib.bj_batch_inverse_ext(self._h, self._ptr(c0), self._ptr(c1), c0.numel()))
        return c0, c1

    def quotening_operation_in_extension(self, acc_c0, acc_c1, sources, values_at, at, challenges):
        """DEEP accumulation for one opening point (cs/implementations/prover.rs:2523-2706).
        sources: list of (c0_tensor, c1_tensor_or_None), each the flat [L*n] LDE of a polynomial."""
        n_src = len(sources)
        p0 = (ctypes.c_void_p * n_src)(*[s[0].data_ptr() for s in sources])
        p1 = (ctypes.c_void_p * n_src)(*[(s[1].data_ptr() if s[1] is not None else None) for s in sources])
        vals = (ctypes.c_uint64 * (2 * n_src))(*[int(x) for v in values_at for x in v])
        chs = (ctypes.c_uint64 * (2 * n_src))(*[int(x) for v in challenges for x in v])
        at_ = (ctypes.c_uint64 * 2)(int(at[0]), int(at[1]))
        log_rows = (acc_c0.numel() * self.shard_world).bit_length() - 1      # global domain size
        self._check(lib.bj_deep_quotient_group(self._h, p0, p1, n_src, vals, chs, at_, log_rows,
                                               self._ptr(acc_c0), self._ptr(acc_c1)))
        return acc_c0, acc_c1

    # ---- stage 2 ----
    @staticmethod
    def non_residues_for_copy_permutation(domain_size, num_columns):
        out = np.zeros(num_columns, np.uint64)
        _ok(lib.bj_non_residues_for_copy_permutation(domain_size, num_columns, out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def compute_partial_products_in_extension(self, variables, sigmas, beta, gamma, max_degree):
        """copy_permutation.rs:649-766.  variables / sigmas: lists of [n] CUDA tensors (natural order).
        Returns (z_c0, z_c1, partials[(c0, c1), ...])."""
        torch = self._torch
        n_cols, n = len(variables), variables[0].numel()
        n_chunks = (n_cols + max_degree - 1) // max_degree
        nr = self.non_residues_for_copy_permutation(n, n_cols)
        pv = (ctypes.c_void_p * n_cols)(*[v.data_ptr() for v in variables])
        ps = (ctypes.c_void_p * n_cols)(*[v.data_ptr() for v in sigmas])
        dev = variables[0].device
        z0 = torch.empty(n, dtype=torch.int64, device=dev)
        z1 = torch.empty(n, dtype=torch.int64, device=dev)
        partials = torch.empty((max(n_chunks - 1, 1), 2, n), dtype=torch.int64, device=dev)
        b = (ctypes.c_uint64 * 2)(int(beta[0]), int(beta[1]))
        g = (ctypes.c_uint64 * 2)(int(gamma[0]), int(gamma[1]))
        self._check(lib.bj_copy_permutation_stage2(self._h, pv, ps, n_cols, nr.ctypes.data_as(ctypes.c_void_p), b, g,
                                                   n.bit_length() - 1, max_degree, self._ptr(z0), self._ptr(z1), self._ptr(partials)))
        return z0, z1, [(partials[c, 0], partials[c, 1]) for c in range(n_chunks - 1)]

    def quotient_copy_permutation(self, var_ldes, sigma_ldes, z, partials, beta, gamma, alphas, log_n, log_lde, log_q, chunk,
                                  q_c0, q_c1):
        """copy-permutation relations + z(1)=1 term on the first 2^log_q cosets (copy_permutation.rs:1000-1249,
        prover.rs:1189-1227).  *_ldes: flat [L*n] CUDA tensors; partials: list of (c0, c1); alphas: n_chunks+1 Fp2."""
        n_cols = len(var_ldes)
        pv = (ctypes.c_void_p * n_cols)(*[v.data_ptr() for v in var_ldes])
        ps = (ctypes.c_void_p * n_cols)(*[v.data_ptr() for v in sigma_ldes])
        flat = [t for pr in partials for t in pr]
        pp = (ctypes.c_void_p * max(1, len(flat)))(*[t.data_ptr() for t in flat])
        nr = self.non_residues_for_copy_permutation(1 << log_n, n_cols)
        b = (ctypes.c_uint64 * 2)(int(beta[0]), int(beta[1]))
        g = (ctypes.c_uint64 * 2)(int(gamma[0]), int(gamma[1]))
        al = (ctypes.c_uint64 * (2 * len(alphas)))(*[int(x) for a in alphas for x in a])
        self._check(lib.bj_quotient_copy_permutation(self._h, pv, ps, n_cols, nr.ctypes.data_as(ctypes.c_void_p),
                                                     self._ptr(z[0]), self._ptr(z[1]), pp, b, g, al, log_n, log_lde, log_q, chunk,
                                                     self._ptr(q_c0), self._ptr(q_c1)))

    def divide_by_vanishing(self, q_c0, q_c1, log_n, log_q):
        self._check(lib.bj_quotient_divide_by_vanishing(self._h, self._ptr(q_c0), self._ptr(q_c1), log_n, log_q))

    def barycentric_evaluate(self, cols, log_n, at):
        """values of base-field polynomials at an Fp2 point from coset 0 of their LDE -> list of (c0, c1)."""
        n_cols = len(cols)
        pc = (ctypes.c_void_p * n_cols)(*[c.data_ptr() for c in cols])
        a = (ctypes.c_uint64 * 2)(int(at[0]), int(at[1]))
        out = np.zeros((n_cols, 2), np.uint64)
        self._check(lib.bj_barycentric_evaluate(self._h, pc, n_cols, log_n, a, out.ctypes.data_as(ctypes.c_void_p)))
        return [(int(r[0]), int(r[1])) for r in out]

    # ---- lookup argument ----
    def compute_lookup_poly_pairs_specialized(self, lookup_cols, width, table_id_col, table_cols, multiplicity, beta, gamma):
        """lookup_argument_in_ext.rs:320-947.  lookup_cols: flat list of n_sub*width [n] tensors.  Returns
        ([(A_i.c0, A_i.c1)], (B.c0, B.c1))."""
        torch = self._torch
        n_sub, n = len(lookup_cols) // width, lookup_cols[0].numel()
        pl = (ctypes.c_void_p * len(lookup_cols))(*[c.data_ptr() for c in lookup_cols])
        pt = (ctypes.c_void_p * len(table_cols))(*[c.data_ptr() for c in table_cols])
        out = torch.empty((n_sub + 1, 2, n), dtype=torch.int64, device=lookup_cols[0].device)
        b = (ctypes.c_uint64 * 2)(int(beta[0]), int(beta[1]))
        g = (ctypes.c_uint64 * 2)(int(gamma[0]), int(gamma[1]))
        self._check(lib.bj_lookup_polys_specialized(self._h, pl, n_sub, width, self._ptr(table_id_col) if table_id_col is not None else None,
                                                    pt, len(table_cols), self._ptr(multiplicity), b, g, n.bit_length() - 1, self._ptr(out)))
        return [(out[i, 0], out[i, 1]) for i in range(n_sub)], (out[n_sub, 0], out[n_sub, 1])

    def quotient_lookup_specialized(self, lookup_ldes, width, table_id_lde, table_ldes, multiplicity_lde, a_ldes, b_lde, beta, gamma,
                                    alphas, q_c0, q_c1):
        n_sub = len(lookup_ldes) // width
        pl = (ctypes.c_void_p * len(lookup_ldes))(*[c.data_ptr() for c in lookup_ldes])
        pt = (ctypes.c_void_p * len(table_ldes))(*[c.data_ptr() for c in table_ldes])
        flat = [t for pr in a_ldes for t in pr]
        pa = (ctypes.c_void_p * len(flat))(*[t.data_ptr() for t in flat])
        b = (ctypes.c_uint64 * 2)(int(beta[0]), int(beta[1]))
        g = (ctypes.c_uint64 * 2)(int(gamma[0]), int(gamma[1]))
        al = (ctypes.c_uint64 * (2 * len(alphas)))(*[int(x) for a in alphas for x in a])
        self._check(lib.bj_quotient_lookup_specialized(self._h, pl, n_sub, width, self._ptr(table_id_lde) if table_id_lde is not None else None,
                                                       pt, len(table_ldes), self._ptr(multiplicity_lde), pa, self._ptr(b_lde[0]),
                                                       self._ptr(b_lde[1]), b, g, al, q_c0.numel(), self._ptr(q_c0), self._ptr(q_c1)))

    # ---- gate / quotient evaluator ----
    def evaluate_gates_over_general_purpose_columns(self, gates, variables, witnesses, constants, alpha_powers, q_c0, q_c1):
        """Row loop of prove_cpu_basic over general-purpose columns (cs/implementations/prover.rs:1031-1080).
        gates: list of dicts {relations: [(op, dst, (kind, value), (kind, value) | None)], writes: [(kind, value)],
        num_repetitions, variables_offset, witnesses_offset, constants_offset, constants_placement_offset,
        selector_path: [bool]} - the data of gpu_synthesizer::GPUDataCapture; columns: lists of flat CUDA tensors."""
        keep, descs = self._gate_descs(gates)

        def ptrs(cols):
            return (ctypes.c_void_p * max(1, len(cols)))(*[c.data_ptr() for c in cols])

        n_terms = len(alpha_powers)
        al = (ctypes.c_uint64 * max(2, 2 * n_terms))(*[int(x) for a in alpha_powers for x in a])
        self._check(lib.bj_quotient_gates_general_purpose(
            self._h, descs, len(gates), ptrs(variables), len(variables), ptrs(witnesses), len(witnesses),
            ptrs(constants), len(constants), al, n_terms, q_c0.numel(), self._ptr(q_c0), self._ptr(q_c1)))
        return q_c0, q_c1

    @staticmethod
    def _gate_descs(gates):
        """list of gate dicts -> (keep-alive list, ctypes array of bj_gate_desc)"""
        N = native
        keep, descs = [], (N.GateDesc * max(1, len(gates)))()
        for d, g in zip(descs, gates):
            rels = (N.GateRelation * max(1, len(g["relations"])))()
            for r, (op, dst, a, b) in zip(rels, g["relations"]):
                r.op, r.dst_temporary = op, dst
                r.a.kind, r.a.value = a[0], int(a[1])
                if b is not None:
                    r.b.kind, r.b.value = b[0], int(b[1])
            wr = (N.GateIndex * max(1, len(g["writes"])))()
            for w, (k, v) in zip(wr, g["writes"]):
                w.kind, w.value = k, int(v)
            path = (ctypes.c_uint8 * max(1, len(g["selector_path"])))(*[int(bool(x)) for x in g["selector_path"]])
            keep += [rels, wr, path]
            d.relations, d.n_relations = rels, len(g["relations"])
            d.writes, d.n_writes = wr, len(g["writes"])
            d.num_repetitions = g["num_repetitions"]
            d.variables_offset, d.witnesses_offset = g.get("variables_offset", 0), g.get("witnesses_offset", 0)
            d.constants_offset = g.get("constants_offset", 0)
            d.constants_placement_offset = g["constants_placement_offset"]
            d.selector_path_len, d.selector_path = len(g["selector_path"]), path
            d.variables_initial_offset, d.witnesses_initial_offset = g.get("variables_initial_offset", 0), g.get("witnesses_initial_offset", 0)
        return keep, descs

    # ---- proof of work ----
    def pow_blake2s(self, seed_bytes, pow_bits):
        """impl PoWRunner for Blake2s256 (cs/implementations/pow.rs:52-147)."""
        seed = (ctypes.c_uint8 * max(1, len(seed_bytes)))(*seed_bytes)
        out = ctypes.c_uint64()
        self._check(lib.bj_pow_blake2s(self._h, seed, len(seed_bytes), pow_bits, ctypes.byref(out)))
        return int(out.value)

    def pow_keccak256(self, seed_bytes, pow_bits):
        """impl PoWRunner for Keccak256 (cs/implementations/pow.rs:140-230)."""
        seed = (ctypes.c_uint8 * max(1, len(seed_bytes)))(*seed_bytes)
        out = ctypes.c_uint64()
        self._check(lib.bj_pow_keccak256(self._h, seed, len(seed_bytes), pow_bits, ctypes.byref(out)))
        return int(out.value)

    # ---- setup / witness materialisation ----
    def materialize_variables_polynomials_from_dense_hint(self, all_values, hint, log_n):
        """witness.rs:325-385.  all_values: [n_values] CUDA tensor; hint: [n_cols, hint_rows] CUDA tensor of reference
        `Variable`s (bit 63 = placeholder).  Returns [n_cols, 2^log_n]."""
        torch = self._torch
        assert hint.is_cuda and hint.is_contiguous() and hint.dim() == 2 and all_values.is_contiguous()
        out = torch.empty((hint.shape[0], 1 << log_n), dtype=torch.int64, device=hint.device)
        self._check(lib.bj_materialize_columns(self._h, self._ptr(all_values), all_values.numel(), self._ptr(hint), hint.shape[0],
                                               hint.shape[1], log_n, self._ptr(out)))
        return out

    def create_permutation_polys(self, placement):
        """setup.rs:419-502.  placement: [n_cols, n] CUDA tensor of `Variable`s (copy_permutation_data) -> sigma columns."""
        assert placement.is_cuda and placement.is_contiguous() and placement.dim() == 2
        out = self._torch.empty_like(placement)
        self._check(lib.bj_create_permutation_polys(self._h, self._ptr(placement), placement.shape[0], placement.shape[1].bit_length() - 1,
                                                    self._ptr(out)))
        return out

    # ---- satisfiability check (bj_check_satisfied / bj_lookup_multiplicities) ----
    def check_if_satisfied(self, variables, sigmas, constants, gates, lookup=None):
        """CSReferenceAssembly::check_if_satisfied (cs/implementations/satisfiability_test.rs:15-353) on the device: gates, copy
        constraints (from sigma alone) and lookups of a witness, exactly.  variables / sigmas [V, n], constants [C, n],
        lookup["tables"] [width + 1, n], lookup["multiplicities"] [n]: contiguous int64 CUDA tensors.  Returns the report as a
        dict (bj_satisfiability_report without its padding); report["satisfied"] is 1 when nothing failed."""
        for t in (variables, sigmas, constants) + ((lookup["tables"], lookup["multiplicities"]) if lookup else ()):
            assert t.is_cuda and t.is_contiguous() and t.dtype == self._torch.int64
        c, keep = _circuit(self, sigmas.shape[1].bit_length() - 1, sigmas.shape[0], constants.shape[0], gates, lookup)
        rep = native.SatisfiabilityReport()
        self._check(lib.bj_check_satisfied(self._h, ctypes.byref(c), self._ptr(sigmas), self._ptr(constants),
                                           self._ptr(lookup["tables"]) if lookup else None, self._ptr(variables),
                                           self._ptr(lookup["multiplicities"]) if lookup else None, ctypes.byref(rep)))
        del keep
        return rep.to_dict()

    def materialize_multiplicities_polynomials(self, variables, constants, lookup):
        """materialize_multiplicities_polynomials (cs/implementations/witness.rs:225-272) on the device: the lookup multiplicity
        column [n] - on the first table row of every distinct content the number of tuples equal to it, 0 elsewhere.  Raises
        BoojumError if a tuple matches no table row."""
        for t in (variables, constants, lookup["tables"]):
            assert t.is_cuda and t.is_contiguous() and t.dtype == self._torch.int64
        n = variables.shape[1]
        c, keep = _circuit(self, n.bit_length() - 1, variables.shape[0], constants.shape[0], [], lookup)
        out = self._torch.empty(n, dtype=self._torch.int64, device=variables.device)
        self._check(lib.bj_lookup_multiplicities(self._h, ctypes.byref(c), self._ptr(constants), self._ptr(lookup["tables"]),
                                                 self._ptr(variables), self._ptr(out)))
        del keep
        return out

    # ---- native prover driver (bj_setup_create / bj_prove: host C++ inside the library) ----
    def native_setup(self, sigmas, constants, gates, quotient_degree, config, lookup=None, public_inputs=()):
        """bj_setup_create.  sigmas [V, n], constants [C, n], lookup["tables"] [width + 1, n]: contiguous int64 CUDA tensors
        (borrowed by the setup: the returned object keeps them alive)."""
        ns = NativeSetup(self, sigmas, constants, gates, quotient_degree, config, lookup, public_inputs)
        self._children.add(ns)
        return ns

    # ---- queries ----
    def query_leaf_elements(self, sources, indices, elems_per_leaf=1):
        n_src = len(sources)
        ptrs = (ctypes.c_void_p * n_src)(*[s.data_ptr() for s in sources])
        idx = np.ascontiguousarray(np.array(indices, dtype=np.uint64))
        out = np.zeros((len(idx), n_src * elems_per_leaf), np.uint64)
        n_leaves = min(int(s.numel()) for s in sources) // elems_per_leaf
        self._check(lib.bj_query_leaf_elements(self._h, ptrs, n_src, elems_per_leaf, n_leaves, idx.ctypes.data_as(ctypes.c_void_p),
                                               len(idx), out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def merkle_paths(self, tree, indices):
        n_leaves = tree.leaf_hashes.shape[0]
        depth = (n_leaves // tree.cap_size).bit_length() - 1
        idx = np.ascontiguousarray(np.array(indices, dtype=np.uint64))
        out = np.zeros((len(idx), max(depth, 1), 4), np.uint64)
        nodes_ptr = self._ptr(tree.nodes) if tree.nodes.numel() else None
        self._check(lib.bj_merkle_paths(self._h, self._ptr(tree.leaf_hashes), nodes_ptr, n_leaves, tree.cap_size,
                                        idx.ctypes.data_as(ctypes.c_void_p), len(idx), out.ctypes.data_as(ctypes.c_void_p)))
        return out[:, :depth, :]

    # ---- FRI ----
    def do_fri(self, transcript, c0, c1, schedule, lde_degree, cap_size, hasher="poseidon2"):
        """do_fri (cs/implementations/fri/mod.rs:49-357): commit phase driven from the host transcript."""
        log_full = c0.numel().bit_length() - 1
        sched = (ctypes.c_uint32 * len(schedule))(*schedule)
        h = ctypes.c_void_p()
        self._check(lib.bj_do_fri_with_hasher(self._h, transcript._h, self._ptr(c0), self._ptr(c1), log_full, sched, len(schedule),
                                              lde_degree.bit_length() - 1, cap_size, {"poseidon2": 0, "blake2s": 1, "keccak256": 2}[hasher], ctypes.byref(h)))
        fo = FriOracles(h, cap_size, (c0, c1))
        self._children.add(fo)
        return fo

    def fri_fold(self, c0, c1, log_fold, alpha, coset_inv):
        """One oracle step (log_fold folds).  Returns (out_c0, out_c1, new_coset_inv)."""
        torch = self._torch
        m = c0.numel()
        log_m = (m * self.shard_world).bit_length() - 1                      # global vector size
        o0 = torch.empty(m >> log_fold, dtype=torch.int64, device=c0.device)
        o1 = torch.empty(m >> log_fold, dtype=torch.int64, device=c0.device)
        al = (ctypes.c_uint64 * 2)(alpha[0], alpha[1])
        ci = ctypes.c_uint64(coset_inv)
        self._check(lib.bj_fri_fold(self._h, self._ptr(c0), self._ptr(c1), log_m, log_fold, al, ctypes.byref(ci),
                                    self._ptr(o0), self._ptr(o1)))
        return o0, o1, int(ci.value)


class Comm:
    """bj_comm: the communicator of the native coset-sharded prover (csrc/comm.cu).  Creating one on a Context declares the
    context's coset shard; native_setup() / NativeSetup.prove() on that context then run sharded and every rank returns the
    same proof.  Transports: NCCL (one process per GPU) or "local" (ranks = threads of one process on one GPU)."""

    def __init__(self, ctx, handle, rank, world, lde_degree):
        self.ctx, self._h, self.rank, self.world = ctx, handle, rank, world
        ctx.shard_rank, ctx.shard_world, ctx.shard_split = rank, world, _shard_split(world, lde_degree)
        ctx._children.add(self)

    @staticmethod
    def unique_id():
        """ncclGetUniqueId (rank 0); hand the 128 bytes to the other ranks by any side channel"""
        buf = (ctypes.c_uint8 * 128)()
        _ok(lib.bj_comm_unique_id(buf), "bj_comm_unique_id")
        return bytes(buf)

    @classmethod
    def nccl(cls, ctx, unique_id, rank, world, lde_degree):
        h = ctypes.c_void_p()
        buf = (ctypes.c_uint8 * 128)(*unique_id)
        ctx._check(lib.bj_comm_create_nccl(ctx._h, buf, rank, world, lde_degree.bit_length() - 1, ctypes.byref(h)))
        return cls(ctx, h, rank, world, lde_degree)

    @classmethod
    def from_torch_distributed(cls, ctx, dist, lde_degree, group=None):
        """one process per GPU launched by torchrun: torch.distributed only carries the 128-byte NCCL unique id"""
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        box = [cls.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0, group=group)
        return cls.nccl(ctx, box[0], rank, world, lde_degree)

    @staticmethod
    def local_group(world):
        g = ctypes.c_void_p()
        _ok(lib.bj_comm_group_create(world, ctypes.byref(g)), "bj_comm_group_create")
        return g

    @staticmethod
    def destroy_local_group(group):
        lib.bj_comm_group_destroy(group)

    @classmethod
    def local(cls, ctx, group, rank, world, lde_degree):
        h = ctypes.c_void_p()
        ctx._check(lib.bj_comm_create_local(ctx._h, group, rank, lde_degree.bit_length() - 1, ctypes.byref(h)))
        return cls(ctx, h, rank, world, lde_degree)

    def all_gather(self, send, recv):
        """device tensors: recv[r] = rank r's send"""
        self.ctx._check(lib.bj_comm_all_gather(self._h, self.ctx._ptr(send), self.ctx._ptr(recv), send.numel()))
        return recv

    def all_gather_host(self, arr):
        a = np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1)
        out = np.zeros((self.world, a.shape[0]), np.uint64)
        self.ctx._check(lib.bj_comm_all_gather_host(self._h, a.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), a.shape[0]))
        return out

    def broadcast_host(self, arr, root=0):
        a = np.ascontiguousarray(arr, dtype=np.uint64)
        self.ctx._check(lib.bj_comm_broadcast_host(self._h, a.ctypes.data_as(ctypes.c_void_p), a.size, root))
        return a

    def close(self):
        if getattr(self, "_h", None):
            lib.bj_comm_destroy(self._h)
            self._h = None
            self.ctx.shard_rank, self.ctx.shard_world, self.ctx.shard_split = 0, 1, 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def proof_memory_plan(log_n, num_variables, num_constants, quotient_degree, config, lookup=None, world=1):
    """bj_proof_memory_plan: device bytes of native_setup + prove at their peak on each of `world` GPUs, counted from the
    shapes (no device needed).  -> dict(resident=bytes, compact=bytes or None, streamed=bytes or None,
    streamed_sharded=bytes or None, recompute=bytes or None), None where the plan does not apply (compact: one GPU with
    quotient degree < LDE factor; streamed: one GPU with quotient degree > LDE factor, bj_proof_memory_plan_streamed;
    streamed_sharded: the streamed plan on each of `world` GPUs, quotient degree > LDE factor,
    bj_proof_memory_plan_streamed_sharded; recompute: one GPU, any quotient degree, bj_proof_memory_plan_recompute, chosen only
    after Context.allow_recompute_plan)."""
    c = native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree = log_n, num_variables, num_constants, quotient_degree
    c.fri_lde_factor, c.merkle_tree_cap_size = config.fri_lde_factor, config.merkle_tree_cap_size
    c.security_level, c.pow_bits = config.security_level, config.pow_bits
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup["width"], lookup["num_repetitions"]
    out = (ctypes.c_uint64 * 2)()
    _ok(lib.bj_proof_memory_plan(ctypes.byref(c), world, out), "bj_proof_memory_plan")
    streamed = ctypes.c_uint64()
    _ok(lib.bj_proof_memory_plan_streamed(ctypes.byref(c), world, ctypes.byref(streamed)), "bj_proof_memory_plan_streamed")
    sharded = ctypes.c_uint64()
    _ok(lib.bj_proof_memory_plan_streamed_sharded(ctypes.byref(c), world, ctypes.byref(sharded)), "bj_proof_memory_plan_streamed_sharded")
    recompute = ctypes.c_uint64()
    _ok(lib.bj_proof_memory_plan_recompute(ctypes.byref(c), world, ctypes.byref(recompute)), "bj_proof_memory_plan_recompute")
    return {"resident": int(out[0]), "compact": int(out[1]) or None, "streamed": int(streamed.value) or None,
            "streamed_sharded": int(sharded.value) or None, "recompute": int(recompute.value) or None}


def proof_memory_plan_recompute_sharded(log_n, num_variables, num_constants, quotient_degree, config, world, lookup=None):
    """bj_proof_memory_plan_recompute_sharded: device bytes of native_setup + prove on each of `world` GPUs on the recompute
    plan, counted from the shapes (no device needed); at world 1 proof_memory_plan()["recompute"].  Chosen only after
    Context.allow_sharded_recompute_plan.  Raises BoojumError for a world sharding rejects (cap_size < world,
    world > 8 * LDE factor, row blocks of fewer than 2 rows)."""
    c = native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree = log_n, num_variables, num_constants, quotient_degree
    c.fri_lde_factor, c.merkle_tree_cap_size = config.fri_lde_factor, config.merkle_tree_cap_size
    c.security_level, c.pow_bits = config.security_level, config.pow_bits
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup["width"], lookup["num_repetitions"]
    out = ctypes.c_uint64()
    _ok(lib.bj_proof_memory_plan_recompute_sharded(ctypes.byref(c), world, ctypes.byref(out)), "bj_proof_memory_plan_recompute_sharded")
    return int(out.value)


def proof_memory_plan_recompute_blocks(log_n, num_variables, num_constants, quotient_degree, config, blocks, lookup=None):
    """bj_proof_memory_plan_recompute_blocks: device bytes of native_setup + prove on one GPU on the recompute plan with every
    coset cut into `blocks` row blocks (1, 2, 4 or 8) in the trees and the quotient, counted from the shapes (no device
    needed); at blocks = 1 proof_memory_plan()["recompute"].  Raises BoojumError for other block counts and for row blocks of
    fewer than 2 rows."""
    c = native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree = log_n, num_variables, num_constants, quotient_degree
    c.fri_lde_factor, c.merkle_tree_cap_size = config.fri_lde_factor, config.merkle_tree_cap_size
    c.security_level, c.pow_bits = config.security_level, config.pow_bits
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup["width"], lookup["num_repetitions"]
    out = ctypes.c_uint64()
    _ok(lib.bj_proof_memory_plan_recompute_blocks(ctypes.byref(c), blocks, ctypes.byref(out)), "bj_proof_memory_plan_recompute_blocks")
    return int(out.value)


def proof_memory_plan_lanes(log_n, num_variables, num_constants, quotient_degree, config, plan, n_lanes, lookup=None, row_blocks=1):
    """bj_proof_memory_plan_lanes_host(_blocks): device bytes of one setup proved on n_lanes lanes at once on one GPU, on `plan`
    ("resident", "compact", "streamed" or "recompute", the last with row_blocks row blocks per coset), counted from the shapes
    (no device needed) -> dict(setup=bytes the setup and the shared tables hold, lane=bytes each lane adds, total=setup +
    n_lanes * lane), or None where the plan does not apply.  At one lane, total is proof_memory_plan()[plan] (and
    proof_memory_plan_recompute_blocks for row_blocks > 1)."""
    c = native.Circuit()
    c.log_n, c.num_variables, c.num_constants, c.quotient_degree = log_n, num_variables, num_constants, quotient_degree
    c.fri_lde_factor, c.merkle_tree_cap_size = config.fri_lde_factor, config.merkle_tree_cap_size
    c.security_level, c.pow_bits = config.security_level, config.pow_bits
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup["width"], lookup["num_repetitions"]
    kind = {"resident": native.PLAN_RESIDENT, "compact": native.PLAN_COMPACT, "streamed": native.PLAN_STREAMED,
            "recompute": native.PLAN_RECOMPUTE}[plan]
    out = (ctypes.c_uint64 * 3)()
    _ok(lib.bj_proof_memory_plan_lanes_host_blocks(ctypes.byref(c), kind, row_blocks, n_lanes, out), "bj_proof_memory_plan_lanes_host_blocks")
    return {"setup": int(out[0]), "lane": int(out[1]), "total": int(out[2])} if out[2] else None


def witness_slots_bytes(log_n, num_variables, n_slots, max_values=0, lookup=None, world=1):
    """bj_witness_slots_bytes: device bytes of a set of n_slots witness slots (with a WitnessVec buffer of max_values values and
    the u32 variables hint when max_values > 0) on each of `world` GPUs, counted from the shapes (no device needed)"""
    c = native.Circuit()
    c.log_n, c.num_variables = log_n, num_variables
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup["width"], lookup["num_repetitions"]
    out = ctypes.c_uint64()
    _ok(lib.bj_witness_slots_bytes(ctypes.byref(c), world, n_slots, max_values, ctypes.byref(out)), "bj_witness_slots_bytes")
    return int(out.value)


def witness_slots_bytes_split(log_n, num_variables, n_slots, max_values=0, lookup=None):
    """bj_witness_slots_bytes_split: witness_slots_bytes at world 1 split in two -> (bytes the set itself allocates in its
    context's pool, bytes of the u32 variables hint, which lives once on the setup: 0 when max_values == 0).  A set on a lane
    (NativeSetup.witness_slots(..., ctx=lane)) counts the first only (no device needed)"""
    c = native.Circuit()
    c.log_n, c.num_variables = log_n, num_variables
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup["width"], lookup["num_repetitions"]
    out = (ctypes.c_uint64 * 2)()
    _ok(lib.bj_witness_slots_bytes_split(ctypes.byref(c), n_slots, max_values, out), "bj_witness_slots_bytes_split")
    return int(out[0]), int(out[1])


def variables_hint_to_u32(hint):
    """bj_variables_hint_to_u32: reference `Variable`s (bit 63 = placeholder) -> (u32 hint with placeholders 0xFFFFFFFF, 1 + the
    largest index).  Raises BoojumError(BJ_ERR_INVALID_ARG) on an index >= 2^32 - 1."""
    h = np.ascontiguousarray(np.asarray(hint).view(np.uint64))
    out = np.empty(h.shape, np.uint32)
    need = ctypes.c_uint64()
    _ok(lib.bj_variables_hint_to_u32(h.ctypes.data_as(ctypes.c_void_p), h.size, out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(need)),
        "bj_variables_hint_to_u32")
    return out, int(need.value)


def _on_device(witness):
    """True for a witness of CUDA tensors, False for host arrays"""
    return bool(getattr(witness[0], "is_cuda", False))


def _host_array(a, dtype, n):
    """(pointer, keep-alive) of a contiguous host array of n elements of dtype: a numpy array or a CPU torch tensor, pinned or
    pageable (a numpy copy is made only when the layout is not already right)"""
    if hasattr(a, "data_ptr"):
        assert not a.is_cuda and a.is_contiguous() and a.element_size() == np.dtype(dtype).itemsize and a.numel() == n
        return ctypes.c_void_p(a.data_ptr()), a
    arr = np.ascontiguousarray(a)
    assert arr.dtype.itemsize == np.dtype(dtype).itemsize and arr.size == n, (arr.dtype, arr.size, n)
    return arr.ctypes.data_as(ctypes.c_void_p), arr


class WitnessSlots:
    """bj_witness_slots: witness slots of one NativeSetup on the device, filled from host memory on the context's copy stream
    while proofs run on its stream.  ctx: the setup's context (the default) or one of its lanes (Context.lane), whose own copy
    stream, pool and stream the set then uses; only that lane's thread may use the set."""

    def __init__(self, setup, n, max_values=0, ctx=None):
        self.setup, self.ctx, self.n, self.max_values = setup, ctx or setup.ctx, n, max_values
        _, self.V, _, _, _, _, lookup, _ = setup._vk_args
        self.lookup = bool(lookup)
        self.rows = 1 << setup._vk_args[0]
        self._held = [[] for _ in range(n)]  # host arrays pending uploads may still read (pinned memory is copied asynchronously)
        h = ctypes.c_void_p()
        self.ctx._check(lib.bj_witness_slots_create(self.ctx._h, setup._h, n, max_values, ctypes.byref(h)))
        self._h = h

    def upload(self, slot, variables, multiplicities=None):
        """bj_witness_upload: variables [V, n] (u64 / int64) and, with a lookup, multiplicities [n]"""
        pv, kv = _host_array(variables, np.uint64, self.V * self.rows)
        pm, km = _host_array(multiplicities, np.uint64, self.rows) if multiplicities is not None else (None, None)
        self.ctx._check(lib.bj_witness_upload(self._h, slot, pv, pm))
        self._held[slot % self.n].append((kv, km))

    def upload_vec(self, slot, all_values, multiplicities=None):
        """bj_witness_upload_vec: WitnessVec.all_values (u64) and WitnessVec.multiplicities (u32), gathered through the hint"""
        nv = len(all_values)
        pv, kv = _host_array(all_values, np.uint64, nv)
        nm = len(multiplicities) if multiplicities is not None else 0
        pm, km = _host_array(multiplicities, np.uint32, nm) if multiplicities is not None else (None, None)
        self.ctx._check(lib.bj_witness_upload_vec(self._h, slot, pv, nv, pm, nm))
        self._held[slot % self.n].append((kv, km))

    def columns(self, slot):
        """bj_witness_slot_columns: a host copy of the slot's columns -> (variables [V, n], multiplicities [n] or None), uint64"""
        d = ctypes.c_void_p()
        self.ctx._check(lib.bj_witness_slot_columns(self._h, slot, ctypes.byref(d)))
        out = np.empty((self.V + self.lookup) * self.rows, np.uint64)
        self.ctx._check(lib.bj_download(self.ctx._h, out.ctypes.data_as(ctypes.c_void_p), d, out.nbytes))
        self.ctx.synchronize()
        v = out[: self.V * self.rows].reshape(self.V, self.rows)
        return v, (out[self.V * self.rows:] if self.lookup else None)

    def prove(self, slot, timings=None, as_json=True):
        """bj_prove_slot: the proof of the slot's witness (same bytes as NativeSetup.prove on it)"""
        h = ctypes.c_void_p()
        self.ctx._check(lib.bj_prove_slot(self.ctx._h, self.setup._h, self._h, slot, ctypes.byref(h)))
        self._held[slot % self.n] = []
        return self.setup._proof_out(h, timings, as_json)

    def close(self):
        if getattr(self, "_h", None):
            lib.bj_witness_slots_free(self._h)
            self._h = None
            self._held = [[] for _ in range(self.n)]

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _circuit(ctx, log_n, num_variables, num_constants, gates, lookup):
    """bj_circuit with the trace shape, the gate programs and the lookup description filled in -> (circuit, keep-alive list)"""
    keep, descs = ctx._gate_descs(gates)
    c = native.Circuit()
    c.log_n, c.num_variables, c.num_constants = log_n, num_variables, num_constants
    c.gates, c.n_gates = descs, len(gates)
    if lookup:
        c.lookup_width, c.lookup_num_repetitions = lookup["width"], lookup["num_repetitions"]
        c.lookup_variables_offset, c.lookup_table_id_column = lookup["variables_offset"], lookup["table_id_column"]
    return c, keep


class NativeSetup:
    """bj_setup: setup LDE + setup tree + circuit description held by the library; prove() runs bj_prove (host C++)."""

    def __init__(self, ctx, sigmas, constants, gates, quotient_degree, config, lookup=None, public_inputs=()):
        import json as _json
        self._json = _json
        self.ctx = ctx
        self._keep = [sigmas, constants, lookup["tables"] if lookup else None]
        for t in self._keep:
            assert t is None or (t.is_cuda and t.is_contiguous() and t.dtype == ctx._torch.int64)
        c, keep = _circuit(ctx, sigmas.shape[1].bit_length() - 1, sigmas.shape[0], constants.shape[0], gates, lookup)
        c.quotient_degree, c.fri_lde_factor, c.merkle_tree_cap_size = quotient_degree, config.fri_lde_factor, config.merkle_tree_cap_size
        c.security_level, c.pow_bits = config.security_level, config.pow_bits
        pis = [(int(a), int(b)) for a, b in public_inputs]
        pc = (ctypes.c_uint32 * max(1, len(pis)))(*[a for a, _ in pis])
        pr = (ctypes.c_uint32 * max(1, len(pis)))(*[b for _, b in pis])
        c.public_input_columns, c.public_input_rows, c.n_public_inputs = pc, pr, len(pis)
        c.tree_hasher = {"poseidon2": 0, "blake2s": 1, "keccak256": 2}[getattr(config, "hasher", "poseidon2")]
        c.transcript = {"poseidon2": 0, "blake2s": 1, "keccak256": 2, "poseidon": 3}[getattr(config, "transcript", "poseidon2")]
        self.cap_size = config.merkle_tree_cap_size
        self._vk_args = (c.log_n, c.num_variables, c.num_constants, gates, quotient_degree, config, lookup, pis)
        h = ctypes.c_void_p()
        ctx._check(lib.bj_setup_create(ctx._h, ctypes.byref(c), ctx._ptr(sigmas), ctx._ptr(constants),
                                       ctx._ptr(lookup["tables"]) if lookup else None, ctypes.byref(h)))
        self._h = h
        del keep

    @property
    def compact(self):
        """True if bj_setup_create chose the compact memory plan"""
        return lib.bj_setup_is_compact(self._h) == 1

    @property
    def plan(self):
        """the memory plan bj_setup_create chose (bj_setup_plan): "resident", "compact", "streamed" or "recompute\""""
        k = lib.bj_setup_plan(self._h)
        _ok(min(k, 0), "bj_setup_plan")
        return {native.PLAN_RESIDENT: "resident", native.PLAN_COMPACT: "compact", native.PLAN_STREAMED: "streamed",
                native.PLAN_RECOMPUTE: "recompute"}[k]

    @property
    def row_blocks(self):
        """the row blocks per coset bj_setup_create chose for the recompute plan on one GPU (bj_setup_row_blocks); 1 on every
        other plan"""
        k = lib.bj_setup_row_blocks(self._h)
        _ok(min(k, 0), "bj_setup_row_blocks")
        return int(k)

    def memory_plan(self):
        """bj_setup_memory_plan: the chosen plan -> dict(pool=peak pool bytes of setup + prove, outside_pool=bound on the
        library's other device memory, chunk=columns the compact or recompute plan recomputes at a time, 0 on the resident and
        streamed plans)"""
        out = (ctypes.c_uint64 * 3)()
        _ok(lib.bj_setup_memory_plan(self._h, out), "bj_setup_memory_plan")
        return {"pool": int(out[0]), "outside_pool": int(out[1]), "chunk": int(out[2])}

    def get_cap(self):
        out = np.zeros((self.cap_size, 4), np.uint64)
        _ok(lib.bj_setup_get_cap(self._h, out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def vk(self):
        """verification-key dict of this setup (same shape as prover.Setup.vk())"""
        from .prover import verification_key
        return verification_key(*self._vk_args, self.get_cap())

    def prove(self, variables, multiplicities=None, timings=None, as_json=False, ctx=None):
        """bj_prove -> the proof as a dict in the reference's serde shape (or the JSON text).  ctx: the setup's context (the
        default) or one of its lanes (Context.lane)."""
        ctx = ctx or self.ctx
        h = ctypes.c_void_p()
        ctx._check(lib.bj_prove(ctx._h, self._h, ctx._ptr(variables),
                                ctx._ptr(multiplicities) if multiplicities is not None else None, ctypes.byref(h)))
        return self._proof_out(h, timings, as_json)

    def memory_plan_lanes(self, n):
        """bj_proof_memory_plan_lanes: the chosen plan split for n lanes proving at once -> dict(setup=bytes the setup and the
        shared tables hold, lane=bytes each lane adds (its pool's high-water mark plus its scratch and parameter arena),
        lane_pool=the pool part of lane, total=setup + n * lane)"""
        out = (ctypes.c_uint64 * 3)()
        _ok(lib.bj_proof_memory_plan_lanes(self._h, n, out), "bj_proof_memory_plan_lanes")
        pool = ctypes.c_uint64()
        _ok(lib.bj_proof_memory_plan_lane_pool(self._h, ctypes.byref(pool)), "bj_proof_memory_plan_lane_pool")
        return {"setup": int(out[0]), "lane": int(out[1]), "total": int(out[2]), "lane_pool": int(pool.value)}

    def attach_variables_hint(self, hint):
        """bj_setup_attach_variables_hint: the DenseVariablesCopyHint [V, hint_rows] (reference `Variable`s, bit 63 =
        placeholder; a host array) kept on the device as u32.  prove_stream then takes witnesses as WitnessVec pairs."""
        h = np.ascontiguousarray(np.asarray(hint).view(np.uint64))
        assert h.ndim == 2 and h.shape[0] == self._vk_args[1]
        self.ctx._check(lib.bj_setup_attach_variables_hint(self._h, h.ctypes.data_as(ctypes.c_void_p), h.shape[1]))
        self.has_hint = True

    has_hint = False

    def witness_slots(self, n=2, max_values=0, ctx=None):
        """bj_witness_slots_create: n (1 to 4) device slots for witnesses of this setup, plus a WitnessVec buffer of max_values
        values when max_values > 0.  ctx: this setup's context (the default) or one of its lanes; prove_stream(..., slots=set)
        then proves on that lane.  Attach the hint before creating sets on lanes."""
        ws = WitnessSlots(self, n, max_values, ctx)
        ws.ctx._children.add(ws)
        return ws

    def prove_stream(self, witnesses, as_json=True, slots=None):
        """Proves a stream of witnesses against this setup, yielding the proofs in order.  witnesses: an iterable of
        (variables [V, n], multiplicities [n] or None) host arrays, or, once a hint is attached, of (all_values,
        multiplicities as u32) WitnessVec pairs.  With N slots (default: a 2-slot set made here) witness k + N - 1 is uploaded,
        on the copy stream, before witness k is proved, so the copy overlaps the proof.  Pinned host arrays are read
        asynchronously and are held until their proof is yielded."""
        own = slots is None
        it = iter(witnesses)
        pending = []
        try:
            first = next(it)
        except StopIteration:
            return
        if own:
            slots = self.witness_slots(2, len(first[0]) if self.has_hint else 0)
        try:
            k = 0
            for w in itertools.chain([first], it):
                s = k % slots.n
                slots.upload(s, *w) if not self.has_hint else slots.upload_vec(s, *w)
                pending.append(s)
                k += 1
                if len(pending) == slots.n:
                    yield slots.prove(pending.pop(0), as_json=as_json)
            while pending:
                yield slots.prove(pending.pop(0), as_json=as_json)
        finally:
            if own:
                slots.close()

    def prove_concurrent(self, witnesses, lanes=2, as_json=True, slots_per_lane=2):
        """Proves several witnesses at once on this setup's GPU, yielding the proofs in input order (each the bytes
        prove() returns).  `lanes` lane contexts (Context.lane) prove them, each from its own thread; the lanes are closed at
        the end, also on an exception.  witnesses: an iterable of
          - (variables [V, n], multiplicities [n] or None) CUDA tensors, complete on the current torch stream when they are
            taken from the iterable, proved from a thread pool, at most two witnesses per lane ahead of the one yielded; or
          - host witnesses: the host arrays prove_stream takes (numpy or CPU torch, pinned or pageable; WitnessVec pairs once
            a hint is attached).  Witness i goes to lane i % lanes, which runs prove_stream over its share through its own
            slot set of `slots_per_lane` slots (uploads on the lane's copy stream overlap its proofs), at most
            lanes * slots_per_lane witnesses ahead of the one yielded.  The slot sets are freed at the end.
        A mix of device and host witnesses raises ValueError: for a list or tuple before any proof, for another iterable when
        the first witness of the other kind is taken."""
        if isinstance(witnesses, (list, tuple)) and len({_on_device(w) for w in witnesses}) > 1:
            raise ValueError("prove_concurrent: the witnesses mix CUDA tensors and host arrays")
        it = iter(witnesses)
        try:
            first = next(it)
        except StopIteration:
            return
        device = _on_device(first)

        def checked():
            for w in itertools.chain([first], it):
                if _on_device(w) != device:
                    raise ValueError("prove_concurrent: the witnesses mix CUDA tensors and host arrays")
                yield w

        if device:
            yield from self._prove_concurrent_device(checked(), lanes, as_json)
        else:
            yield from self._prove_concurrent_host(checked(), len(first[0]) if self.has_hint else 0, lanes, as_json, slots_per_lane)

    def _prove_concurrent_device(self, witnesses, lanes, as_json):
        import collections
        import queue
        from concurrent.futures import ThreadPoolExecutor
        torch = self.ctx._torch
        ctxs = [self.ctx.lane() for _ in range(lanes)]
        idle = queue.Queue()
        for c in ctxs:
            idle.put(c)

        def one(w):
            c = idle.get()
            try:
                return self.prove(w[0], w[1] if len(w) > 1 else None, as_json=as_json, ctx=c)
            finally:
                idle.put(c)

        pool = ThreadPoolExecutor(max_workers=lanes)
        try:
            pending = collections.deque()
            for w in witnesses:
                torch.cuda.current_stream(self.ctx.device).synchronize()  # the lanes' streams do not wait for torch's
                pending.append(pool.submit(one, w))
                if len(pending) >= 2 * lanes:
                    yield pending.popleft().result()
            while pending:
                yield pending.popleft().result()
        finally:
            pool.shutdown(wait=True, cancel_futures=True)
            for c in ctxs:
                c.close()

    def _prove_concurrent_host(self, witnesses, max_values, lanes, as_json, slots_per_lane):
        import queue
        import threading
        end = object()
        stop = threading.Event()
        inbox = [queue.Queue() for _ in range(lanes)]
        outbox = [queue.Queue() for _ in range(lanes)]
        ctxs, sets, threads = [], [], []

        def lane_main(k):
            def feed():
                while not stop.is_set():
                    w = inbox[k].get()
                    if w is end:
                        return
                    yield w
            try:
                for p in self.prove_stream(feed(), as_json=as_json, slots=sets[k]):
                    outbox[k].put((True, p))
            except BaseException as e:  # noqa: BLE001 - raised on the caller's thread
                outbox[k].put((False, e))

        def result(i):
            ok, v = outbox[i % lanes].get()
            if not ok:
                raise v
            return v

        try:
            for _ in range(lanes):
                ctxs.append(self.ctx.lane())
                sets.append(self.witness_slots(slots_per_lane, max_values, ctx=ctxs[-1]))
            threads = [threading.Thread(target=lane_main, args=(k,), daemon=True) for k in range(lanes)]
            for t in threads:
                t.start()
            # a lane yields witness i's proof once it holds slots_per_lane - 1 later witnesses (or the end): those are
            # queued before the proof is awaited
            ahead = lanes * slots_per_lane
            taken = done = 0
            for w in witnesses:
                inbox[taken % lanes].put(w)
                taken += 1
                if taken - done >= ahead:
                    yield result(done)
                    done += 1
            for q in inbox:
                q.put(end)
            while done < taken:
                yield result(done)
                done += 1
        finally:
            stop.set()
            for q in inbox:
                q.put(end)
            for t in threads:
                t.join()
            for ws in sets:
                ws.close()
            for c in ctxs:
                c.close()

    def _proof_out(self, h, timings, as_json):
        """a bj_proof handle -> the proof as a dict or JSON text (the handle is freed)"""
        try:
            need = ctypes.c_size_t()
            _ok(lib.bj_proof_to_json(h, None, 0, ctypes.byref(need)))
            buf = ctypes.create_string_buffer(need.value)
            _ok(lib.bj_proof_to_json(h, buf, need.value, ctypes.byref(need)))
            if timings is not None:
                st = (ctypes.c_double * 6)()
                _ok(lib.bj_proof_stage_seconds(h, st))
                for k, v in zip(("1_witness_lde_commit", "2_stage2_products_lde_commit", "3_quotient", "4_openings", "5_deep_fri", "6_queries"), st):
                    timings[k] = float(v)
        finally:
            lib.bj_proof_free(h)
        text = buf.value.decode()
        return text if as_json else self._json.loads(text)

    def close(self):
        if getattr(self, "_h", None):
            lib.bj_setup_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
