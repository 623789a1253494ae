"""ctypes binding of libboojum_b200.so (the C-ABI in include/boojum_b200.h).

This is the only way Python reaches the kernels: there is no Python or CPU fallback.  If the shared library
has not been built (`python -c "import __graft_entry__ as g; g.build()"` or `make -C era_boojum_b200`) the import
of this module raises.  PyTorch is used by callers for device memory and streams only; this module
itself only needs ctypes.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_VARIANT = os.environ.get("BJ_LIB_VARIANT")   # debugging / A-B builds: libboojum_b200_<variant>.so
LIB_PATH = os.path.join(_HERE, "libboojum_b200_%s.so" % _VARIANT if _VARIANT else "libboojum_b200.so")

P = 0xFFFFFFFF00000001

BJ_OK = 0
BJ_ERR_INVALID_ARG = -1
BJ_ERR_CUDA = -2
BJ_ERR_NO_DEVICE = -3
BJ_ERR_OOM = -4
BJ_ERR_UNSUPPORTED = -5


class BoojumError(RuntimeError):
    def __init__(self, status, message):
        super().__init__("boojum_b200 status %d: %s" % (status, message))
        self.status = status


if not os.path.exists(LIB_PATH):
    raise ImportError(
        "era_boojum_b200: %s is missing - build it with `make -C era_boojum_b200` (nvcc, sm_90a). "
        "There is no CPU fallback." % LIB_PATH)

lib = ctypes.CDLL(LIB_PATH)

_u64, _u32, _i32, _sz, _vp = ctypes.c_uint64, ctypes.c_uint32, ctypes.c_int32, ctypes.c_size_t, ctypes.c_void_p
_pp = ctypes.POINTER(ctypes.c_void_p)

SIGNATURES = {
    "bj_version": (ctypes.c_char_p, []),
    "bj_status_string": (ctypes.c_char_p, [_i32]),
    "bj_ctx_create": (_i32, [_i32, _vp, _pp]),
    "bj_ctx_destroy": (_i32, [_vp]),
    "bj_ctx_set_stream": (_i32, [_vp, _vp]),
    "bj_ctx_set_coset_shard": (_i32, [_vp, _u32, _u32, _u32]),
    "bj_ctx_set_domain_shard": (_i32, [_vp, _u32, _u32, _u32]),
    "bj_ctx_synchronize": (_i32, [_vp]),
    "bj_last_error": (ctypes.c_char_p, [_vp]),
    "bj_launch_count": (_u64, [_vp]),
    "bj_ctx_set_memory_limit": (_i32, [_vp, _u64]),
    "bj_ctx_allow_recompute_plan": (_i32, [_vp, _i32]),
    "bj_ctx_allow_sharded_recompute_plan": (_i32, [_vp, _i32]),
    "bj_ctx_set_max_row_blocks": (_i32, [_vp, _u32]),
    "bj_ctx_memory_high_water": (_i32, [_vp, _vp, _i32]),
    "bj_ctx_create_lane": (_i32, [_vp, _pp]),
    "bj_alloc": (_i32, [_vp, _sz, _pp]),
    "bj_free": (_i32, [_vp, _vp]),
    "bj_upload": (_i32, [_vp, _vp, _vp, _sz]),
    "bj_download": (_i32, [_vp, _vp, _vp, _sz]),
    "bj_alloc_host_pinned": (_i32, [_sz, _pp]),
    "bj_free_host_pinned": (_i32, [_vp]),
    "bj_twiddles": (_i32, [_vp, _u32, _i32, _vp]),
    "bj_ntt_natural_to_bitreversed": (_i32, [_vp, _vp, _u32, _u32, _u64, _u64]),
    "bj_intt_natural_to_natural": (_i32, [_vp, _vp, _u32, _u32, _u64, _u64]),
    "bj_bitreverse": (_i32, [_vp, _vp, _u32, _u32, _u64]),
    "bj_lde": (_i32, [_vp, _vp, _u64, _vp, _u32, _u32, _u32, _i32]),
    "bj_lde_next_row": (_i32, [_vp, _vp, _u64, _vp, _u32, _u32, _u32, _i32]),
    "bj_lde_cosets": (_i32, [_vp, _vp, _u64, _vp, _u32, _u32, _u32, _u32, _u32, _i32]),
    "bj_merkle_build_poseidon2": (_i32, [_vp, _vp, _u32, _u64, _u32, _u32, _vp, _vp]),
    "bj_merkle_build_blake2s": (_i32, [_vp, _vp, _u32, _u64, _u32, _u32, _vp, _vp]),
    "bj_merkle_build_keccak256": (_i32, [_vp, _vp, _u32, _u64, _u32, _u32, _vp, _vp]),
    "bj_poseidon2_hash_rows": (_i32, [_vp, _vp, _u64, _u32, _vp]),
    "bj_poseidon2_permute": (_i32, [_vp, _vp, _u64]),
    "bj_fri_fold": (_i32, [_vp, _vp, _vp, _u32, _u32, _vp, _vp, _vp, _vp]),
    "bj_batch_inverse": (_i32, [_vp, _vp, _u64]),
    "bj_batch_inverse_ext": (_i32, [_vp, _vp, _vp, _u64]),
    "bj_deep_quotient_group": (_i32, [_vp, _vp, _vp, _u32, _vp, _vp, _vp, _u32, _vp, _vp]),
    "bj_deep_quotient_range": (_i32, [_vp, _vp, _vp, _u32, _vp, _vp, _vp, _u32, _u64, _u64, _vp, _vp]),
    "bj_non_residues_for_copy_permutation": (_i32, [_u64, _u32, _vp]),
    "bj_copy_permutation_stage2": (_i32, [_vp, _vp, _vp, _u32, _vp, _vp, _vp, _u32, _u32, _vp, _vp, _vp]),
    "bj_quotient_copy_permutation": (_i32, [_vp, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _u32, _u32, _vp, _vp]),
    "bj_quotient_copy_permutation_with_z_next": (_i32, [_vp, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _u32, _u32, _vp, _vp]),
    "bj_quotient_divide_by_vanishing": (_i32, [_vp, _vp, _vp, _u32, _u32]),
    "bj_barycentric_evaluate": (_i32, [_vp, _vp, _u32, _u32, _vp, _vp]),
    "bj_lookup_polys_specialized": (_i32, [_vp, _vp, _u32, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _u32, _vp]),
    "bj_quotient_lookup_specialized": (_i32, [_vp, _vp, _u32, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp]),
    "bj_quotient_gates_general_purpose": (_i32, [_vp, _vp, _u32, _vp, _u32, _vp, _u32, _vp, _u32, _vp, _u32, _u64, _vp, _vp]),
    "bj_gate_programs_compile": (_i32, [_vp, _u32, _u32, _u32, _u32, _u32, _vp, _u64, _vp, _vp, _vp]),
    "bj_ntt_natural_to_bitreversed_host": (_i32, [_vp, _vp, _u32, _u32, _u64]),
    "bj_intt_natural_to_natural_host": (_i32, [_vp, _vp, _u32, _u32, _u64]),
    "bj_transcript_new": (_vp, []),
    "bj_transcript_new_blake2s": (_vp, []),
    "bj_transcript_new_keccak256": (_vp, []),
    "bj_transcript_new_poseidon": (_vp, []),
    "bj_transcript_free": (None, [_vp]),
    "bj_transcript_witness_field_elements": (None, [_vp, _vp, _sz]),
    "bj_transcript_witness_merkle_tree_cap": (None, [_vp, _vp, _sz]),
    "bj_transcript_get_challenge": (_u64, [_vp]),
    "bj_transcript_get_index_bits": (_u64, [_vp, _u32, _u32]),
    "bj_compute_fri_schedule": (_i32, [_u32, _u32, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp]),
    "bj_do_fri": (_i32, [_vp, _vp, _vp, _vp, _u32, _vp, _u32, _u32, _u32, _pp]),
    "bj_do_fri_with_hasher": (_i32, [_vp, _vp, _vp, _vp, _u32, _vp, _u32, _u32, _u32, _u32, _pp]),
    "bj_fri_oracles_free": (None, [_vp]),
    "bj_fri_oracles_num_oracles": (_u32, [_vp]),
    "bj_fri_oracles_num_monomials": (_u32, [_vp]),
    "bj_fri_oracles_get_cap": (_i32, [_vp, _u32, _vp]),
    "bj_fri_oracles_get_monomials": (_i32, [_vp, _vp, _vp]),
    "bj_fri_oracles_get_challenges": (_i32, [_vp, _vp]),
    "bj_fri_oracles_query": (_i32, [_vp, _u32, _u64, _vp, _vp, _vp]),
    "bj_fri_oracles_query_batch": (_i32, [_vp, _u32, _vp, _u32, _vp, _vp, _vp]),
    "bj_query_leaf_elements": (_i32, [_vp, _vp, _u32, _u32, _u64, _vp, _u32, _vp]),
    "bj_merkle_paths": (_i32, [_vp, _vp, _vp, _u64, _u32, _vp, _u32, _vp]),
    "bj_pow_blake2s": (_i32, [_vp, _vp, _u32, _u32, _vp]),
    "bj_pow_keccak256": (_i32, [_vp, _vp, _u32, _u32, _vp]),
    "bj_materialize_columns": (_i32, [_vp, _vp, _u64, _vp, _u32, _u64, _u32, _vp]),
    "bj_create_permutation_polys": (_i32, [_vp, _vp, _u32, _u32, _vp]),
    "bj_comm_unique_id": (_i32, [_vp]),
    "bj_comm_create_nccl": (_i32, [_vp, _vp, _u32, _u32, _u32, _pp]),
    "bj_comm_group_create": (_i32, [_u32, _pp]),
    "bj_comm_group_destroy": (None, [_vp]),
    "bj_comm_create_local": (_i32, [_vp, _vp, _u32, _u32, _pp]),
    "bj_comm_destroy": (_i32, [_vp]),
    "bj_comm_rank": (_u32, [_vp]),
    "bj_comm_world": (_u32, [_vp]),
    "bj_comm_all_gather": (_i32, [_vp, _vp, _vp, _u64]),
    "bj_comm_all_gather_host": (_i32, [_vp, _vp, _vp, _u64]),
    "bj_comm_broadcast_host": (_i32, [_vp, _vp, _u64, _u32]),
    "bj_setup_create": (_i32, [_vp, _vp, _vp, _vp, _vp, _pp]),
    "bj_setup_free": (None, [_vp]),
    "bj_proof_memory_plan": (_i32, [_vp, _u32, _vp]),
    "bj_proof_memory_plan_streamed": (_i32, [_vp, _u32, _vp]),
    "bj_proof_memory_plan_streamed_sharded": (_i32, [_vp, _u32, _vp]),
    "bj_proof_memory_plan_recompute": (_i32, [_vp, _u32, _vp]),
    "bj_proof_memory_plan_recompute_sharded": (_i32, [_vp, _u32, _vp]),
    "bj_proof_memory_plan_recompute_blocks": (_i32, [_vp, _u32, _vp]),
    "bj_setup_is_compact": (_i32, [_vp]),
    "bj_setup_plan": (_i32, [_vp]),
    "bj_setup_row_blocks": (_i32, [_vp]),
    "bj_setup_memory_plan": (_i32, [_vp, _vp]),
    "bj_proof_memory_plan_lanes": (_i32, [_vp, _u32, _vp]),
    "bj_proof_memory_plan_lane_pool": (_i32, [_vp, _vp]),
    "bj_proof_memory_plan_lanes_host": (_i32, [_vp, _u32, _u32, _vp]),
    "bj_proof_memory_plan_lanes_host_blocks": (_i32, [_vp, _u32, _u32, _u32, _vp]),
    "bj_setup_get_cap": (_i32, [_vp, _vp]),
    "bj_prove": (_i32, [_vp, _vp, _vp, _vp, _pp]),
    "bj_proof_free": (None, [_vp]),
    "bj_proof_to_json": (_i32, [_vp, _vp, _sz, ctypes.POINTER(_sz)]),
    "bj_proof_stage_seconds": (_i32, [_vp, _vp]),
    "bj_witness_slots_bytes": (_i32, [_vp, _u32, _u32, _u64, _vp]),
    "bj_witness_slots_bytes_split": (_i32, [_vp, _u32, _u64, _vp]),
    "bj_witness_slots_create": (_i32, [_vp, _vp, _u32, _u64, _pp]),
    "bj_witness_slots_free": (None, [_vp]),
    "bj_witness_upload": (_i32, [_vp, _u32, _vp, _vp]),
    "bj_setup_attach_variables_hint": (_i32, [_vp, _vp, _u64]),
    "bj_variables_hint_to_u32": (_i32, [_vp, _u64, _vp, _vp]),
    "bj_witness_upload_vec": (_i32, [_vp, _u32, _vp, _u64, _vp, _u64]),
    "bj_prove_slot": (_i32, [_vp, _vp, _vp, _u32, _pp]),
    "bj_witness_slot_columns": (_i32, [_vp, _u32, _pp]),
    "bj_check_satisfied": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bj_lookup_multiplicities": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "bj_selftest_field": (_i32, [_vp, _u64, _u64, _vp]),
    "bj_host_gl_mul": (_u64, [_u64, _u64]),
    "bj_host_gl_add": (_u64, [_u64, _u64]),
    "bj_host_gl_sub": (_u64, [_u64, _u64]),
    "bj_host_gl_inv": (_u64, [_u64]),
    "bj_host_gl_mul_pow2": (_u64, [_u64, _u32]),
    "bj_host_e2_mul": (None, [_vp, _vp, _vp]),
    "bj_host_e2_inv": (None, [_vp, _vp]),
    "bj_host_poseidon2_permutation": (None, [_vp]),
    "bj_host_poseidon_permutation": (None, [_vp]),
    "bj_host_keccak256": (None, [_vp, _sz, _vp]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)  # AttributeError here == header/library mismatch
    _fn.restype = _res
    _fn.argtypes = _args


def version():
    return lib.bj_version().decode()


class GateIndex(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("value", ctypes.c_uint64)]


class GateRelation(ctypes.Structure):
    _fields_ = [("op", ctypes.c_uint32), ("dst_temporary", ctypes.c_uint32), ("a", GateIndex), ("b", GateIndex)]


class GateDesc(ctypes.Structure):
    _fields_ = [("relations", ctypes.POINTER(GateRelation)), ("n_relations", ctypes.c_uint32), ("n_writes", ctypes.c_uint32),
                ("writes", ctypes.POINTER(GateIndex)), ("num_repetitions", ctypes.c_uint32),
                ("variables_offset", ctypes.c_uint32), ("witnesses_offset", ctypes.c_uint32),
                ("constants_offset", ctypes.c_uint32), ("constants_placement_offset", ctypes.c_uint32),
                ("selector_path_len", ctypes.c_uint32), ("selector_path", ctypes.POINTER(ctypes.c_uint8)),
                ("variables_initial_offset", ctypes.c_uint32), ("witnesses_initial_offset", ctypes.c_uint32)]


PLAN_RESIDENT, PLAN_COMPACT, PLAN_STREAMED, PLAN_RECOMPUTE = range(4)  # BJ_PLAN_*
IDX_VARIABLE, IDX_WITNESS, IDX_CONSTANT_POLY, IDX_TEMPORARY, IDX_CONSTANT_VALUE, IDX_CONSTANT_POLY_SHARED = range(6)
REL_ADD, REL_DOUBLE, REL_SUB, REL_NEGATE, REL_MUL, REL_SQUARE, REL_INVERSE = range(7)


class Circuit(ctypes.Structure):
    """bj_circuit"""
    _fields_ = [("log_n", ctypes.c_uint32), ("num_variables", ctypes.c_uint32), ("num_constants", ctypes.c_uint32),
                ("quotient_degree", ctypes.c_uint32), ("fri_lde_factor", ctypes.c_uint32), ("merkle_tree_cap_size", ctypes.c_uint32),
                ("security_level", ctypes.c_uint32), ("pow_bits", ctypes.c_uint32), ("gates", ctypes.POINTER(GateDesc)),
                ("n_gates", ctypes.c_uint32), ("lookup_width", ctypes.c_uint32), ("lookup_num_repetitions", ctypes.c_uint32),
                ("lookup_variables_offset", ctypes.c_uint32), ("lookup_table_id_column", ctypes.c_uint32),
                ("public_input_columns", ctypes.POINTER(ctypes.c_uint32)), ("public_input_rows", ctypes.POINTER(ctypes.c_uint32)),
                ("n_public_inputs", ctypes.c_uint32), ("tree_hasher", ctypes.c_uint32), ("transcript", ctypes.c_uint32)]


SIGMA_NO_CELL, SIGMA_UNNAMED, SIGMA_NAMED_TWICE = 1, 2, 3


class SatisfiabilityReport(ctypes.Structure):
    """bj_satisfiability_report"""
    _fields_ = [("satisfied", ctypes.c_uint32), ("reserved0", ctypes.c_uint32),
                ("gate_failures", ctypes.c_uint64), ("gate_row", ctypes.c_uint64), ("gate_index", ctypes.c_uint32),
                ("gate_repetition", ctypes.c_uint32), ("gate_term", ctypes.c_uint32), ("reserved1", ctypes.c_uint32),
                ("gate_value", ctypes.c_uint64), ("gate_selector", ctypes.c_uint64),
                ("copy_failures", ctypes.c_uint64), ("copy_row", ctypes.c_uint64), ("copy_other_row", ctypes.c_uint64),
                ("copy_column", ctypes.c_uint32), ("copy_other_column", ctypes.c_uint32),
                ("copy_value", ctypes.c_uint64), ("copy_other_value", ctypes.c_uint64),
                ("sigma_failures", ctypes.c_uint64), ("sigma_row", ctypes.c_uint64), ("sigma_column", ctypes.c_uint32),
                ("sigma_kind", ctypes.c_uint32),
                ("lookup_unmatched", ctypes.c_uint64), ("lookup_row", ctypes.c_uint64), ("lookup_subargument", ctypes.c_uint32),
                ("reserved2", ctypes.c_uint32),
                ("multiplicity_failures", ctypes.c_uint64), ("multiplicity_row", ctypes.c_uint64),
                ("multiplicity_count", ctypes.c_uint64), ("multiplicity_sum", ctypes.c_uint64)]

    def to_dict(self):
        """the report without its padding fields"""
        return {name: int(getattr(self, name)) for name, _ in self._fields_ if not name.startswith("reserved")}
