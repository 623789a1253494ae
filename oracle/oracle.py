"""ORACLE (test infrastructure, NOT product code): ctypes/numpy front-end of oracle/liboracle.so.

Each wrapper names the reference function it restates (paths relative to src/ of the era-boojum repository).
All arrays are numpy uint64, canonical Goldilocks values on output.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

P = 0xFFFFFFFF00000001
MULT_GEN = 7


def build(force=False):
    """Compile oracle/liboracle.so with the system gcc (oracle/Makefile).  make runs every time and rebuilds the library
    when a source is newer, so a library built from an older oracle.c (one that lacks symbols lib() looks up) is not
    loaded; an up-to-date library is left alone, so a read-only tree works once it is built."""
    subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        u64, sz, vp = ctypes.c_uint64, ctypes.c_size_t, ctypes.c_void_p
        sig = {
            "orc_add": (u64, [u64, u64]), "orc_sub": (u64, [u64, u64]), "orc_mul": (u64, [u64, u64]),
            "orc_mul_slow": (u64, [u64, u64]), "orc_inv": (u64, [u64]), "orc_pow": (u64, [u64, u64]),
            "orc_omega": (u64, [ctypes.c_uint]),
            "orc_ext_mul": (None, [vp, vp, vp]), "orc_ext_inv": (None, [vp, vp]),
            "orc_num_threads": (ctypes.c_int, []), "orc_set_threads": (None, [ctypes.c_int]),
            "orc_bitreverse": (None, [vp, ctypes.c_uint]),
            "orc_twiddles": (None, [vp, ctypes.c_uint, ctypes.c_int, ctypes.c_int]),
            "orc_ntt_n2b": (None, [vp, ctypes.c_uint, sz, sz, u64]),
            "orc_intt_n2n": (None, [vp, ctypes.c_uint, sz, sz, u64]),
            "orc_lde": (None, [vp, vp, ctypes.c_uint, ctypes.c_uint, sz, ctypes.c_int]),
            "orc_naive_dft_bitreversed": (None, [vp, vp, ctypes.c_uint, u64]),
            "orc_poseidon2_permutation": (None, [vp]),
            "orc_poseidon2_hash_leaf": (None, [vp, sz, vp]),
            "orc_poseidon2_hash_node": (None, [vp, vp, vp]),
            "orc_merkle_leaf_hashes": (None, [vp, sz, sz, sz, vp]),
            "orc_merkle_nodes": (sz, [vp, sz, sz, vp]),
            "orc_merkle_verify": (ctypes.c_int, [vp, vp, sz, vp, sz, sz]),
            "orc_fri_fold": (None, [vp, vp, sz, vp, vp, u64, vp, vp]),
            "orc_batch_inverse": (None, [vp, sz]),
            "orc_batch_inverse_ext": (None, [vp, vp, sz]),
            "orc_deep_point": (None, [vp, vp, vp, vp, vp, vp, vp, sz, u64, vp]),
            "orc_deep_group": (None, [vp, vp, vp, vp, sz, vp, vp, vp, ctypes.c_uint]),
            "orc_cp_stage2": (None, [vp, vp, sz, vp, vp, vp, ctypes.c_uint, sz, vp, vp, vp, vp]),
            "orc_cp_quotient": (None, [vp, vp, sz, vp, vp, vp, vp, vp, vp, vp, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint, sz,
                                       vp, vp]),
            "orc_divide_by_vanishing": (None, [vp, vp, ctypes.c_uint, ctypes.c_uint]),
            "orc_lookup_polys": (None, [vp, sz, sz, vp, vp, sz, vp, vp, vp, sz, vp]),
            "orc_lookup_quotient": (None, [vp, sz, sz, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp, sz, vp, vp]),
            "orc_horner_ext": (None, [vp, sz, sz, vp, vp]),
            "orc_gates_quotient": (None, [vp, sz, vp, vp, vp, ctypes.c_uint32, ctypes.c_uint32, vp, sz, vp, vp]),
            "orc_gates_check": (None, [vp, sz, vp, vp, vp, ctypes.c_uint32, sz, vp, vp, vp]),
            "orc_materialize_columns": (u64, [vp, sz, vp, sz, sz, ctypes.c_uint, vp]),
            "orc_create_permutation_polys": (ctypes.c_int, [vp, sz, ctypes.c_uint, vp, vp]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---------------------------------------------------------------- field -----
def add(a, b):
    return lib().orc_add(a, b)


def sub(a, b):
    return lib().orc_sub(a, b)


def mul(a, b):
    return lib().orc_mul(a, b)


def inv(a):
    return lib().orc_inv(a)


def pow_(a, e):
    return lib().orc_pow(a, e)


def omega(log_n):
    """domain_generator_for_size (cs/implementations/utils.rs:13-28)."""
    return lib().orc_omega(log_n)


def ext_mul(a, b):
    x, y, o = _u64(a), _u64(b), np.zeros(2, np.uint64)
    lib().orc_ext_mul(_p(x), _p(y), _p(o))
    return (int(o[0]), int(o[1]))


def ext_inv(a):
    x, o = _u64(a), np.zeros(2, np.uint64)
    lib().orc_ext_inv(_p(x), _p(o))
    return (int(o[0]), int(o[1]))


def set_threads(n):
    lib().orc_set_threads(n)


def num_threads():
    return lib().orc_num_threads()


# ------------------------------------------------------------------ NTT -----
def bitreverse(a):
    a = _u64(a).copy()
    log_n = int(a.shape[-1]).bit_length() - 1
    flat = a.reshape(-1, a.shape[-1])
    for row in flat:
        lib().orc_bitreverse(_p(row), log_n)
    return a


def twiddles(log_n, inverse=False, with_assert=False):
    """precompute_twiddles_for_fft (cs/implementations/utils.rs:88-125)."""
    t = np.zeros(max(1, (1 << log_n) // 2), np.uint64)
    lib().orc_twiddles(_p(t), log_n, int(inverse), int(with_assert))
    return t


def ntt_n2b(cols, coset=1):
    """fft_natural_to_bitreversed per column (fft/mod.rs:398-411); cols: [n_cols, n] or [n]."""
    a = _u64(cols).copy()
    n = a.shape[-1]
    ncols = a.size // n
    lib().orc_ntt_n2b(_p(a), n.bit_length() - 1, ncols, n, coset)
    return a


def intt_n2n(cols, coset=1):
    """ifft_natural_to_natural per column (fft/mod.rs:464-491)."""
    a = _u64(cols).copy()
    n = a.shape[-1]
    ncols = a.size // n
    lib().orc_intt_n2n(_p(a), n.bit_length() - 1, ncols, n, coset)
    return a


def lde(cols, log_lde, from_monomials=False):
    """transform_raw_storages_to_lde (cs/implementations/utils.rs:270-403) -> [n_cols, L, n]."""
    a = _u64(cols)
    if a.ndim == 1:
        a = a[None, :]
    ncols, n = a.shape
    out = np.zeros((ncols, 1 << log_lde, n), np.uint64)
    lib().orc_lde(_p(a), _p(out), n.bit_length() - 1, log_lde, ncols, int(from_monomials))
    return out


def naive_dft_bitreversed(a, coset=1):
    a = _u64(a)
    out = np.zeros_like(a)
    lib().orc_naive_dft_bitreversed(_p(a), _p(out), a.shape[0].bit_length() - 1, coset)
    return out


# ------------------------------------------------------------ Poseidon2 -----
def poseidon2_permutation(state):
    s = _u64(state).copy()
    assert s.shape == (12,)
    lib().orc_poseidon2_permutation(_p(s))
    return s


def poseidon2_hash_leaf(els):
    e, o = _u64(els), np.zeros(4, np.uint64)
    lib().orc_poseidon2_hash_leaf(_p(e), e.shape[0], _p(o))
    return o


def poseidon2_hash_node(l, r):
    a, b, o = _u64(l), _u64(r), np.zeros(4, np.uint64)
    lib().orc_poseidon2_hash_node(_p(a), _p(b), _p(o))
    return o


def merkle_leaf_hashes(sources, elems_per_leaf=1):
    """sources: list of flat uint64 arrays (each n_leaves*elems_per_leaf long), in leaf-preimage order."""
    srcs = [_u64(s).reshape(-1) for s in sources]
    n_leaves = srcs[0].shape[0] // elems_per_leaf
    ptrs = (ctypes.c_void_p * len(srcs))(*[s.ctypes.data for s in srcs])
    out = np.zeros((n_leaves, 4), np.uint64)
    lib().orc_merkle_leaf_hashes(ptrs, len(srcs), n_leaves, elems_per_leaf, _p(out))
    return out


def merkle_nodes(leaf_hashes, cap_size):
    """continue_from_leaf_hashes (cs/oracle/merkle_tree.rs:388-449): list of levels (bottom-up)."""
    lh = _u64(leaf_hashes)
    n = lh.shape[0]
    total = max(0, n - cap_size)
    nodes = np.zeros((max(total, 1), 4), np.uint64)
    w = lib().orc_merkle_nodes(_p(lh), n, cap_size, _p(nodes))
    assert w == total
    levels, off, cnt = [], 0, n
    while cnt > cap_size:
        cnt //= 2
        levels.append(nodes[off:off + cnt])
        off += cnt
    return levels


def merkle_tree(sources, cap_size, elems_per_leaf=1):
    lh = merkle_leaf_hashes(sources, elems_per_leaf)
    levels = merkle_nodes(lh, cap_size)
    cap = levels[-1] if levels else lh
    return lh, levels, cap


def merkle_path(lh, levels, idx):
    """get_proof (cs/oracle/merkle_tree.rs:462-480): siblings bottom-up, cap level excluded."""
    path = []
    layers = [lh] + list(levels[:-1]) if levels else []
    for layer in layers:
        path.append(layer[idx ^ 1].copy())
        idx >>= 1
    return np.array(path, dtype=np.uint64).reshape(-1, 4)


def merkle_verify(leaf_hash, path, cap, idx):
    lh, pa, ca = _u64(leaf_hash), _u64(path).reshape(-1, 4), _u64(cap).reshape(-1, 4)
    return bool(lib().orc_merkle_verify(_p(lh), _p(pa), pa.shape[0], _p(ca), ca.shape[0], idx))


# ------------------------------------------------------------------ FRI -----
def fri_fold(c0, c1, alpha, roots, coset_inv):
    """fold_multiple (cs/implementations/fri/mod.rs:362-474), one fold-by-2."""
    a, b, r = _u64(c0), _u64(c1), _u64(roots)
    al = _u64(alpha)
    m = a.shape[0]
    o0, o1 = np.zeros(m // 2, np.uint64), np.zeros(m // 2, np.uint64)
    lib().orc_fri_fold(_p(a), _p(b), m, _p(al), _p(r), coset_inv, _p(o0), _p(o1))
    return o0, o1


def batch_inverse(a):
    x = _u64(a).copy()
    lib().orc_batch_inverse(_p(x), x.shape[0])
    return x


def batch_inverse_ext(c0, c1):
    x, y = _u64(c0).copy(), _u64(c1).copy()
    lib().orc_batch_inverse_ext(_p(x), _p(y), x.shape[0])
    return x, y


def deep_point(acc, f, v, ch, x, at):
    """One quotening_operation group at one point (verifier.rs:2526-2565).  f, v, ch: lists of (c0,c1)."""
    f, v, ch = _u64(f).reshape(-1, 2), _u64(v).reshape(-1, 2), _u64(ch).reshape(-1, 2)
    cols = [np.ascontiguousarray(t[:, k]) for t in (f, v, ch) for k in (0, 1)]
    a, at_ = _u64(acc).copy(), _u64(at)
    lib().orc_deep_point(_p(a), *[_p(c) for c in cols], f.shape[0], x, _p(at_))
    return (int(a[0]), int(a[1]))


def deep_group(acc0, acc1, sources, values_at, challenges, at):
    """quotening_operation_in_extension over the whole LDE domain (prover.rs:2523-2706).
    sources: list of (c0_array, c1_array_or_None); returns updated (acc0, acc1)."""
    a0, a1 = _u64(acc0).copy(), _u64(acc1).copy()
    c0s = [_u64(s[0]).reshape(-1) for s in sources]
    c1s = [(_u64(s[1]).reshape(-1) if s[1] is not None else None) for s in sources]
    n = len(sources)
    p0 = (ctypes.c_void_p * n)(*[c.ctypes.data for c in c0s])
    p1 = (ctypes.c_void_p * n)(*[(c.ctypes.data if c is not None else None) for c in c1s])
    vals = _u64(np.array(values_at, dtype=np.uint64).reshape(-1))
    chs = _u64(np.array(challenges, dtype=np.uint64).reshape(-1))
    at_ = _u64(np.array(at, dtype=np.uint64))
    lib().orc_deep_group(_p(a0), _p(a1), p0, p1, n, _p(vals), _p(chs), _p(at_), a0.shape[0].bit_length() - 1)
    return a0, a1


# ----------------------------------------------------------- copy permutation / lookup / openings -----
def _ptrs(cols):
    """list of 1-D uint64 arrays -> (ctypes pointer array, contiguous arrays kept alive by the caller)"""
    arrs = [_u64(c).reshape(-1) for c in cols]
    return (ctypes.c_void_p * max(1, len(arrs)))(*[a.ctypes.data for a in arrs]), arrs


def _e2(v):
    return _u64(np.array([int(v[0]), int(v[1])], dtype=np.uint64))


def cp_stage2(variables, sigmas, non_residues, beta, gamma, chunk):
    """compute_partial_products_in_extension (cs/implementations/copy_permutation.rs:649-766).  variables / sigmas: lists of
    [n] columns (natural order).  Returns (z_c0, z_c1, partials [n_chunks - 1, 2, n], grand product (c0, c1))."""
    n_cols, n = len(variables), _u64(variables[0]).shape[0]
    n_chunks = (n_cols + chunk - 1) // chunk
    pv, kv = _ptrs(variables)
    ps, ks_ = _ptrs(sigmas)
    ks = _u64(non_residues)
    z0, z1 = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    partials = np.zeros((max(n_chunks - 1, 1), 2, n), np.uint64)
    grand = np.zeros(2, np.uint64)
    lib().orc_cp_stage2(pv, ps, n_cols, _p(ks), _p(_e2(beta)), _p(_e2(gamma)), n.bit_length() - 1, chunk, _p(z0), _p(z1),
                        _p(partials), _p(grand))
    return z0, z1, partials[:n_chunks - 1], (int(grand[0]), int(grand[1]))


def cp_quotient(var_ldes, sigma_ldes, non_residues, z, partials, beta, gamma, alphas, log_n, log_lde, log_q, chunk, q0, q1):
    """copy-permutation quotient terms and the z(1) = 1 term (copy_permutation.rs:1000-1249, prover.rs:1189-1227) on the
    first 2^log_q cosets, added to (q0, q1).  *_ldes, z, partials: flat [L * n] LDE columns; partials: list of (c0, c1)."""
    pv, kv = _ptrs(var_ldes)
    ps, ks_ = _ptrs(sigma_ldes)
    pp, kp = _ptrs([t for pr in partials for t in pr])
    z0, z1 = _u64(z[0]).reshape(-1), _u64(z[1]).reshape(-1)
    al = _u64(np.array(alphas, dtype=np.uint64).reshape(-1))
    ks = _u64(non_residues)
    o0, o1 = _u64(q0).copy(), _u64(q1).copy()
    lib().orc_cp_quotient(pv, ps, len(var_ldes), _p(ks), _p(z0), _p(z1), pp, _p(_e2(beta)), _p(_e2(gamma)), _p(al), log_n,
                          log_lde, log_q, chunk, _p(o0), _p(o1))
    return o0, o1


def divide_by_vanishing(q0, q1, log_n, log_q):
    """divide_by_vanishing_for_bitreversed_coset_enumeration (cs/implementations/utils.rs:770-817)."""
    o0, o1 = _u64(q0).copy(), _u64(q1).copy()
    assert o0.shape[0] == 1 << (log_n + log_q)
    lib().orc_divide_by_vanishing(_p(o0), _p(o1), log_n, log_q)
    return o0, o1


def lookup_polys(lookup_cols, width, table_id_col, table_cols, multiplicity, beta, gamma):
    """compute_lookup_poly_pairs_specialized (cs/implementations/lookup_argument_in_ext.rs:320-947).  lookup_cols: n_sub * width
    columns.  Returns [n_sub + 1, 2, n]: A_0 .. A_{n_sub - 1}, then B."""
    n_sub = len(lookup_cols) // width
    pl, kl = _ptrs(lookup_cols)
    pt, kt = _ptrs(table_cols)
    tid = _u64(table_id_col) if table_id_col is not None else None
    m = _u64(multiplicity)
    n = m.shape[0]
    out = np.zeros((n_sub + 1, 2, n), np.uint64)
    lib().orc_lookup_polys(pl, n_sub, width, _p(tid) if tid is not None else None, pt, len(table_cols), _p(m), _p(_e2(beta)),
                           _p(_e2(gamma)), n, _p(out))
    return out


def lookup_quotient(lookup_ldes, width, table_id_lde, table_ldes, multiplicity_lde, a_ldes, b_lde, beta, gamma, alphas, q0, q1):
    """compute_quotient_terms_for_lookup_specialized (lookup_argument_in_ext.rs:949-1319) at the points of (q0, q1), added to
    them.  a_ldes: list of (c0, c1); b_lde: (c0, c1)."""
    n_sub = len(lookup_ldes) // width
    pl, kl = _ptrs(lookup_ldes)
    pt, kt = _ptrs(table_ldes)
    pa, ka = _ptrs([t for pr in a_ldes for t in pr])
    tid = _u64(table_id_lde).reshape(-1) if table_id_lde is not None else None
    m, b0, b1 = _u64(multiplicity_lde).reshape(-1), _u64(b_lde[0]).reshape(-1), _u64(b_lde[1]).reshape(-1)
    al = _u64(np.array(alphas, dtype=np.uint64).reshape(-1))
    o0, o1 = _u64(q0).copy(), _u64(q1).copy()
    lib().orc_lookup_quotient(pl, n_sub, width, _p(tid) if tid is not None else None, pt, len(table_ldes), _p(m), pa, _p(b0),
                              _p(b1), _p(_e2(beta)), _p(_e2(gamma)), _p(al), o0.shape[0], _p(o0), _p(o1))
    return o0, o1


def horner_ext(monomials, at):
    """f(at) for each row of [n_cols, n] base-field coefficients (low degree first) at an Fp2 point -> [n_cols, 2]."""
    m = _u64(monomials)
    if m.ndim == 1:
        m = m[None, :]
    out = np.zeros((m.shape[0], 2), np.uint64)
    lib().orc_horner_ext(_p(m), m.shape[0], m.shape[1], _p(_e2(at)), _p(out))
    return out


def random_field(rng, shape):
    """Uniform canonical Goldilocks elements from a numpy Generator (rejection below p)."""
    a = rng.integers(0, 2**64, size=shape, dtype=np.uint64)
    bad = a >= np.uint64(P)
    while bad.any():
        a[bad] = rng.integers(0, 2**64, size=int(bad.sum()), dtype=np.uint64)
        bad = a >= np.uint64(P)
    return a


# ------------------------------------------------------------------------------------------ gate programs -----
_GD_WORDS = 13


def _gate_arrays(gates):
    """gate dicts (the form Context.evaluate_gates_over_general_purpose_columns takes) -> the flat descriptor, relation and
    write arrays of orc_gates_quotient / orc_gates_check"""
    desc, rels, writes = [], [], []
    for g in gates:
        path = g["selector_path"]
        assert len(path) <= 32
        desc.append([len(rels), len(g["relations"]), len(writes), len(g["writes"]), g["num_repetitions"], g.get("variables_offset", 0),
                     g.get("witnesses_offset", 0), g.get("constants_offset", 0), g["constants_placement_offset"], len(path),
                     sum(1 << i for i, bit in enumerate(path) if bit), g.get("variables_initial_offset", 0),
                     g.get("witnesses_initial_offset", 0)])
        for op, dst, a, b in g["relations"]:
            b = b if b is not None else (4, 0)
            rels.append([op, dst, a[0], int(a[1]), b[0], int(b[1])])
        writes += [[k, int(v)] for k, v in g["writes"]]
    return (_u64(np.array(desc, dtype=np.uint64).reshape(-1, _GD_WORDS)), _u64(np.array(rels, dtype=np.uint64).reshape(-1, 6)),
            _u64(np.array(writes, dtype=np.uint64).reshape(-1, 2)))


def gates_quotient(gates, variables, witnesses, constants, alphas, q0, q1):
    """q + sum_g sel_g * sum_k alpha_k term_k at every point: what bj_quotient_gates_general_purpose computes, from the recorded
    programs.  variables / witnesses / constants: lists of [n] columns or [cols, n] arrays (lazy u64); alphas: (c0, c1) per
    term.  Returns canonical (q0, q1)."""
    d, r, w = _gate_arrays(gates)
    cols = list(variables) + list(witnesses) + list(constants)
    pc, keep = _ptrs(cols)
    al = _u64(np.array(alphas, dtype=np.uint64).reshape(-1))
    o0, o1 = _u64(q0).copy(), _u64(q1).copy()
    assert al.shape[0] >= 2 * sum(len(g["writes"]) * g["num_repetitions"] for g in gates)
    assert all(c.shape[0] >= o0.shape[0] for c in keep)
    lib().orc_gates_quotient(_p(d), len(gates), _p(r), _p(w), pc, len(variables), len(witnesses), _p(al), o0.shape[0], _p(o0), _p(o1))
    return o0, o1


def gates_check(gates, variables, constants):
    """The gate half of bj_check_satisfied over the rows of the columns: dict(failures, row, term = first failing global term
    index, first_value [n], first_selector [n] - the first failing term's value and its gate's selector per row, 0 on passing
    rows)."""
    d, r, w = _gate_arrays(gates)
    pc, keep = _ptrs(list(variables) + list(constants))
    n = keep[0].shape[0]
    fv, fs, out = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(3, np.uint64)
    lib().orc_gates_check(_p(d), len(gates), _p(r), _p(w), pc, len(variables), n, _p(fv), _p(fs), _p(out))
    return dict(failures=int(out[0]), row=int(out[1]), term=int(out[2]), first_value=fv, first_selector=fs)


def gates_report(gates, variables, constants):
    """gates_check in the fields of bj_satisfiability_report: gate_failures, gate_row, gate_index, gate_repetition, gate_term,
    gate_value, gate_selector (all 0 without failures)"""
    c = gates_check(gates, variables, constants)
    rep = dict(gate_failures=c["failures"], gate_row=0, gate_index=0, gate_repetition=0, gate_term=0, gate_value=0, gate_selector=0)
    if c["failures"]:
        t, base = c["term"], 0
        for gi, g in enumerate(gates):
            size = len(g["writes"]) * g["num_repetitions"]
            if t < base + size:
                break
            base += size
        row = c["row"]
        rep.update(gate_row=row, gate_index=gi, gate_repetition=(t - base) // len(g["writes"]), gate_term=(t - base) % len(g["writes"]),
                   gate_value=int(c["first_value"][row]), gate_selector=int(c["first_selector"][row]))
    return rep


# ------------------------------------------------------------- setup / witness columns -----
def materialize_columns(all_values, hint, log_n):
    """materialize_variables_polynomials_from_dense_hint (cs/implementations/witness.rs:325-385).  all_values [n_values],
    hint [n_cols, hint_rows] of `Variable`s (bit 63 = placeholder) -> (columns [n_cols, 2^log_n], number of non-placeholder
    cells whose index is past all_values; those cells stay 0)."""
    v, h = _u64(all_values), _u64(hint)
    out = np.empty((h.shape[0], 1 << log_n), np.uint64)
    bad = lib().orc_materialize_columns(_p(v), v.size, _p(h), h.shape[0], h.shape[1], log_n, _p(out))
    return out, int(bad)


def create_permutation_polys(placement):
    """create_permutation_polys (cs/implementations/setup.rs:419-502).  placement [n_cols, n] of `Variable`s
    (copy_permutation_data) -> the sigma columns [n_cols, n]."""
    from .stage2 import non_residues_for_copy_permutation
    pl = _u64(placement)
    n_cols, n = pl.shape
    nr = _u64(non_residues_for_copy_permutation(n, n_cols))
    out = np.empty((n_cols, n), np.uint64)
    if lib().orc_create_permutation_polys(_p(pl), n_cols, n.bit_length() - 1, _p(nr), _p(out)):
        raise MemoryError("orc_create_permutation_polys: the scratch table does not fit in host memory")
    return out
