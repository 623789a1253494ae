"""Synthetic SHA-256-bench-shaped circuit (workload generator for tests and bench.py; there is no Rust toolchain here
to synthesise the real circuit, SURVEY.md 8d).

Geometry of the reference bench (src/gadgets/sha256/mod.rs:307-373): 60 general-purpose columns under copy permutation,
gates ConstantsAllocator (4 repetitions), FmaGateInBaseFieldWithoutConstant (15) and ReductionGate<4> (12) selected per
row through a binary selector tree in the first constant columns, quotient degree 4; with lookup=True also the bench's 8
lookup sub-arguments of width 4 over specialised columns (table id in a constant column), and add_specialized_fma() places
extra gates on specialised columns.  Every row satisfies the gate its selector picks, and neighbouring
repetitions of a row are tied by copy constraints (the output of repetition k-1 is an input of repetition k), so the
sigma polynomials are a non-trivial permutation.  All values are kept small enough that plain 64-bit integer arithmetic
is exact, so the trace can be generated with torch on the GPU without field multiplications; the identity permutation
k_j * omega^i comes from the library's own NTT.
"""
import numpy as np

from . import native

N = native
_V, _C, _T, _CS = N.IDX_VARIABLE, N.IDX_CONSTANT_POLY, N.IDX_TEMPORARY, N.IDX_CONSTANT_POLY_SHARED

# GPUDataCapture-style programs (src/gpu_synthesizer/mod.rs:354-443) of the three evaluators
FMA = dict(name="fma", relations=[(N.REL_MUL, 0, (_V, 2), (_CS, 1)), (N.REL_MUL, 1, (_V, 0), (_V, 1)), (N.REL_MUL, 2, (_CS, 0), (_T, 1)),
                                  (N.REL_ADD, 3, (_T, 0), (_T, 2)), (N.REL_SUB, 4, (_T, 3), (_V, 3))],
           writes=[(_T, 4)], variables_offset=4, constants_offset=0)
REDUCTION4 = dict(name="reduction4",
                  relations=[(N.REL_MUL, 0, (_V, 0), (_CS, 0)), (N.REL_MUL, 1, (_V, 1), (_CS, 1)), (N.REL_ADD, 2, (_T, 0), (_T, 1)),
                             (N.REL_MUL, 3, (_V, 2), (_CS, 2)), (N.REL_ADD, 4, (_T, 2), (_T, 3)), (N.REL_MUL, 5, (_V, 3), (_CS, 3)),
                             (N.REL_ADD, 6, (_T, 4), (_T, 5)), (N.REL_SUB, 7, (_T, 6), (_V, 4))],
                  writes=[(_T, 7)], variables_offset=5, constants_offset=0)
CONSTANT_ALLOCATOR = dict(name="constant_allocator", relations=[(N.REL_SUB, 0, (_V, 0), (_C, 0))], writes=[(_T, 0)],
                          variables_offset=1, constants_offset=1)


def sha_shaped_gates(num_variables=60):
    """gate list in registration order with repetitions for `num_variables` columns and a 3-leaf selector tree."""
    def g(base, reps, path):
        d = dict(base)
        d.update(num_repetitions=reps, constants_placement_offset=len(path), selector_path=path)
        return d
    return [g(CONSTANT_ALLOCATOR, min(4, num_variables), [True, True]), g(FMA, num_variables // 4, [True, False]),
            g(REDUCTION4, num_variables // 5, [False])]


def _witness_rnd(rnd, dev, witness_seed):
    """the draw of the free witness values: from the circuit's own generator, or, with a witness seed, from a second one - so
    circuits of one seed and different witness seeds share sigmas, constants and tables (one setup, many witnesses)"""
    if witness_seed is None:
        return rnd
    import torch
    gen = torch.Generator(device=dev)
    gen.manual_seed(witness_seed)
    return lambda shape, hi: torch.randint(0, hi, shape, dtype=torch.int64, device=dev, generator=gen)


def generate(ctx, log_n, num_variables=60, seed=0, lookup=False, witness_seed=None):
    """Returns (variables [V, n], sigmas [V, n], constants [C, n], gates, quotient_degree) as int64 CUDA tensors, C = 6.
    With lookup=True (the bench's 8 sub-arguments of width 4 with a shared table id in a constant column,
    src/gadgets/sha256/mod.rs:340-346): V grows by 32 specialised lookup columns, C = 7 (column 6 = table id) and a sixth
    return value dict(width, num_repetitions, variables_offset, table_id_column, tables [5, n], multiplicities [n]).
    witness_seed: draw the free witness values from their own generator (see _witness_rnd)."""
    torch = ctx._torch
    n_gp = num_variables
    V, n, C = num_variables, 1 << log_n, 6
    dev = "cuda:%d" % ctx.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    rnd = lambda shape, hi: torch.randint(0, hi, shape, dtype=torch.int64, device=dev, generator=gen)
    wrnd = _witness_rnd(rnd, dev, witness_seed)
    gates = sha_shaped_gates(V)
    n_fma, n_red = V // 4, V // 5
    kind = rnd((n,), 3)                     # 0 = constant allocator, 1 = fma, 2 = reduction
    is_ca, is_fma, is_red = kind == 0, kind == 1, kind == 2
    variables = wrnd((V, n), 1 << 20)
    constants = torch.zeros((C, n), dtype=torch.int64, device=dev)
    # selector tree: column 0 splits {reduction | others}, column 1 splits {fma | constant allocator}
    constants[0] = (~is_red).to(torch.int64)
    # ---- fma rows: d_k = c0 * a_k * b_k + c1 * c_k, c1 = 1, c_k = d_{k-1}
    c0 = rnd((n,), 1 << 10) + 1
    fma = wrnd((V, n), 1 << 20)
    for k in range(n_fma):
        if k > 0:
            fma[4 * k + 2] = fma[4 * k - 1]
        fma[4 * k + 3] = c0 * fma[4 * k] * fma[4 * k + 1] + fma[4 * k + 2]
    # ---- reduction rows: r_k = sum_i c_i * v_{k,i}, v_{k,0} = r_{k-1}
    rc = rnd((4, n), 1 << 8)
    rc[0] = 1                               # the chained input enters with coefficient 1 so values grow additively
    red = wrnd((V, n), 1 << 16)
    for k in range(n_red):
        if k > 0:
            red[5 * k] = red[5 * k - 1]
        red[5 * k + 4] = sum(rc[i] * red[5 * k + i] for i in range(4))
    # ---- constant allocator rows: variable r = constant at column 2 + r
    cc = rnd((4, n), 1 << 30)
    variables = torch.where(is_fma[None, :], fma, variables)
    variables = torch.where(is_red[None, :], red, variables)
    n_ca = min(4, V)
    variables[:n_ca] = torch.where(is_ca[None, :], cc[:n_ca], variables[:n_ca])
    # constants per row type
    constants[1] = torch.where(is_red, rc[0], is_ca.to(torch.int64))       # reduction: its 1st constant; else selector bit
    constants[2] = torch.where(is_red, rc[1], torch.where(is_fma, c0, cc[0]))
    constants[3] = torch.where(is_red, rc[2], torch.where(is_fma, torch.ones_like(c0), cc[1]))
    constants[4] = torch.where(is_red, rc[3], torch.where(is_ca, cc[2], torch.zeros_like(c0)))
    constants[5] = torch.where(is_ca, cc[3], torch.zeros_like(c0))
    # ---- sigmas: identity k_j * omega^i from the library NTT of the polynomial k_j * X, then swap the tied cells
    ks = ctx.non_residues_for_copy_permutation(n, V)
    mono = torch.zeros((V, n), dtype=torch.int64, device=dev)
    if n > 1:
        mono[:, 1] = torch.from_numpy(ks.view(np.int64)).to(dev)
    else:
        mono[:, 0] = torch.from_numpy(ks.view(np.int64)).to(dev)
    ctx.fft_natural_to_bitreversed(mono, 1)
    ctx.bitreverse_enumeration_inplace(mono)
    ident = mono
    sigmas = ident.clone()
    for k in range(1, n_fma):
        a, b = 4 * k + 2, 4 * k - 1
        sigmas[a] = torch.where(is_fma, ident[b], sigmas[a])
        sigmas[b] = torch.where(is_fma, ident[a], sigmas[b])
    for k in range(1, n_red):
        a, b = 5 * k, 5 * k - 1
        sigmas[a] = torch.where(is_red, ident[b], sigmas[a])
        sigmas[b] = torch.where(is_red, ident[a], sigmas[b])
    if not lookup:
        return variables.contiguous(), sigmas.contiguous(), constants.contiguous(), gates, 4
    # ---- lookup argument: every row looks up 8 random entries of one width-4 table (table id 1)
    width, nsub = 4, 8
    T = min(n, 1 << 16)
    tables = torch.zeros((width + 1, n), dtype=torch.int64, device=dev)
    idx = torch.arange(T, dtype=torch.int64, device=dev)
    tables[0, :T] = idx
    tables[1, :T] = idx * idx + 3
    tables[2, :T] = idx ^ 0x5555
    tables[3, :T] = 7 * idx + 1
    tables[4, :T] = 1                      # table id column
    picks = wrnd((nsub, n), T)
    lk_cols = torch.stack([tables[j][picks[i]] for i in range(nsub) for j in range(width)])      # [32, n]
    mult = torch.bincount(picks.reshape(-1), minlength=n).to(torch.int64)
    table_id_const = torch.ones((1, n), dtype=torch.int64, device=dev)
    variables = torch.cat([variables, lk_cols], dim=0)
    constants = torch.cat([constants, table_id_const], dim=0)
    # identity sigmas for the lookup columns
    Vt = n_gp + nsub * width
    ks = ctx.non_residues_for_copy_permutation(n, Vt)
    mono = torch.zeros((Vt, n), dtype=torch.int64, device=dev)
    mono[:, 1 if n > 1 else 0] = torch.from_numpy(ks.view(np.int64)).to(dev)
    ctx.fft_natural_to_bitreversed(mono, 1)
    ctx.bitreverse_enumeration_inplace(mono)
    # the first n_gp non-residues are a prefix of the longer list, so the gp sigmas computed above stay valid
    sigmas = torch.cat([sigmas, mono[n_gp:]], dim=0)
    lk = dict(width=width, num_repetitions=nsub, variables_offset=n_gp, table_id_column=6, tables=tables.contiguous(),
              multiplicities=mult.contiguous())
    return variables.contiguous(), sigmas.contiguous(), constants.contiguous(), gates, 4, lk


def add_specialized_fma(ctx, variables, sigmas, constants, gates, repetitions=2, seed=0):
    """Places `repetitions` FMA gates on SPECIALISED columns (GatePlacementStrategy::UseSpecializedColumns with
    share_constants = true, src/cs/implementations/prover.rs:653-801): 4 * repetitions extra variable columns that satisfy
    d = c0 * a * b + c1 * c on EVERY row (no selector), two extra constant columns shared by the repetitions.  The gate is
    put first in the gate list, as the reference orders the quotient terms (specialised before general purpose)."""
    torch = ctx._torch
    V0, n = variables.shape
    C0 = constants.shape[0]
    dev = variables.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(1000 + seed)
    rnd = lambda shape, hi: torch.randint(0, hi, shape, dtype=torch.int64, device=dev, generator=gen)
    c0, c1 = rnd((n,), 1 << 10) + 1, rnd((n,), 1 << 10)
    cols = rnd((4 * repetitions, n), 1 << 20)
    for k in range(repetitions):
        cols[4 * k + 3] = c0 * cols[4 * k] * cols[4 * k + 1] + c1 * cols[4 * k + 2]
    Vt = V0 + 4 * repetitions
    ks = ctx.non_residues_for_copy_permutation(n, Vt)
    mono = torch.zeros((Vt, n), dtype=torch.int64, device=dev)
    mono[:, 1 if n > 1 else 0] = torch.from_numpy(ks.view(np.int64)).to(dev)
    ctx.fft_natural_to_bitreversed(mono, 1)
    ctx.bitreverse_enumeration_inplace(mono)
    g = dict(FMA)
    g.update(name="fma", num_repetitions=repetitions, constants_placement_offset=C0, selector_path=[], variables_initial_offset=V0)
    return (torch.cat([variables, cols]).contiguous(), torch.cat([sigmas, mono[V0:]]).contiguous(),
            torch.cat([constants, torch.stack([c0, c1])]).contiguous(), [g] + list(gates))


# ------------------------------------------------------------------------------------------- production-shaped circuit -----
# Selector tree of the reference's own vk.json (src/gadgets/recursion/recursive_verifier.rs:2281-2368; the fixture under
# tests/golden): gate index in registration order -> TreeNode::output_placement path (left = True).
PRODUCTION_SELECTOR_PATHS = [
    [False, False, False],                          # 0 ConstantsAllocatorGate
    [False, True, True, False, True, True],         # 1 U8x4FMAGate
    [True],                                         # 2 Poseidon2FlattenedGate (130 columns, ~9.6k relations, 118 terms)
    [False, True, True, True, False, True],         # 3 DotProductGate<4>
    [False, True, True, True, False, False],        # 4 ZeroCheckGate
    [False, True, True, True, True],                # 5 FmaGateInBaseFieldWithoutConstant
    [False, True, False],                           # 6 UIntXAddGate
    [False, True, True, False, False, True],        # 7 SelectionGate
    [False, True, True, False, True, False],        # 8 ParallelSelectionGate<4>
    [False, True, True, False, False, False],       # 9 NopGate / PublicInputGate
    [False, False, True],                           # 10 ReductionGate<4>
]


def generate_production_shaped(ctx, log_n, seed=0, witness_seed=None):
    """A circuit with the GEOMETRY of the reference's vk.json / proof.json fixture (a zkSync recursion-layer circuit): 130
    general-purpose columns with the 11 evaluators above behind its 6-level selector tree, 8 lookup sub-arguments of width 3
    over specialised columns (table id in constant column 7), a BooleanConstraintGate on one specialised column - 155 columns
    under the copy permutation, 8 constant columns, quotient degree 8 (to be proven with fri_lde_factor 2, cap 32) - and 4
    public inputs.  Rows are NopGate rows (any values), ConstantsAllocator rows, FMA rows and Reduction rows (chained by copy
    constraints, as in generate()); the other evaluators are selected on no row but are EVALUATED on every point, which is
    what the prover's cost depends on.  Returns dict(variables, sigmas, constants, gates, quotient_degree, lookup,
    public_inputs).  witness_seed: draw the free witness values from their own generator (see _witness_rnd)."""
    from . import gate_library as GL
    torch = ctx._torch
    GP, W, NSUB = 130, 3, 8
    V, C, n = GP + W * NSUB + 1, 8, 1 << log_n
    dev = "cuda:%d" % ctx.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    rnd = lambda shape, hi: torch.randint(0, hi, shape, dtype=torch.int64, device=dev, generator=gen)
    wrnd = _witness_rnd(rnd, dev, witness_seed)
    gp_gates = [GL.CONSTANT_ALLOCATOR, GL.U8X4_FMA, GL.poseidon2_flattened_gate(GP, 0), GL.DOT_PRODUCT4, GL.ZERO_CHECK, GL.FMA,
                GL.UINTX_ADD, GL.SELECTION, GL.PARALLEL_SELECTION4, GL.NOP, GL.REDUCTION4]
    # specialised-column gates come first in the quotient (prover.rs:608-625), then the general-purpose ones in registration order
    gates = [GL.placed(GL.BOOLEAN, 1, [], constants_placement_offset=C, variables_initial_offset=V - 1)]
    for gate, path in zip(gp_gates, PRODUCTION_SELECTOR_PATHS):
        if gate.terms:
            gates.append(GL.placed(gate, gate.num_repetitions_in_geometry(GP, 0, 4), path))
    n_fma, n_red, n_ca = GP // 4, GP // 5, 4
    kind = rnd((n,), 4)                     # 0 = nop, 1 = constants allocator, 2 = fma, 3 = reduction
    is_ca, is_fma, is_red = kind == 1, kind == 2, kind == 3
    gp = wrnd((GP, n), 1 << 20)
    c0 = rnd((n,), 1 << 10) + 1
    fma = wrnd((GP, n), 1 << 20)
    for k in range(n_fma):                  # d_k = c0 * a_k * b_k + 1 * c_k, c_k = d_{k-1}
        if k > 0:
            fma[4 * k + 2] = fma[4 * k - 1]
        fma[4 * k + 3] = c0 * fma[4 * k] * fma[4 * k + 1] + fma[4 * k + 2]
    rc = rnd((4, n), 1 << 8)
    rc[0] = 1
    red = wrnd((GP, n), 1 << 16)
    for k in range(n_red):                  # r_k = sum_i c_i * v_{k,i}, v_{k,0} = r_{k-1}
        if k > 0:
            red[5 * k] = red[5 * k - 1]
        red[5 * k + 4] = sum(rc[i] * red[5 * k + i] for i in range(4))
    cc = rnd((n_ca, n), 1 << 30)
    gp = torch.where(is_fma[None, :], fma, gp)
    gp = torch.where(is_red[None, :], red, gp)
    gp[:n_ca] = torch.where(is_ca[None, :], cc, gp[:n_ca])
    one, zero = torch.ones_like(c0), torch.zeros_like(c0)
    # constant columns: the selected gate's path bits, then that gate's own constants (they start at column len(path))
    pick = lambda nop, ca, fm, rd: torch.where(is_ca, ca, torch.where(is_fma, fm, torch.where(is_red, rd, nop)))
    constants = torch.stack([
        pick(zero, zero, zero, zero),       # column 0: every one of the four paths starts with False
        pick(one, zero, one, zero),         # column 1
        pick(one, zero, one, one),          # column 2
        pick(zero, cc[0], one, rc[0]),      # column 3: nop F | allocator constant 0 | fma path T | reduction coefficient 0
        pick(zero, cc[1], one, rc[1]),      # column 4
        pick(zero, cc[2], c0, rc[2]),       # column 5: fma's row-shared constants start at its path length 5
        pick(zero, cc[3], one, rc[3]),      # column 6
        one,                                # column 7: lookup table id
    ])
    # lookups: every row looks up 8 random entries of one width-3 table (table id 1)
    T = min(n, 1 << 16)
    tables = torch.zeros((W + 1, n), dtype=torch.int64, device=dev)
    idx = torch.arange(T, dtype=torch.int64, device=dev)
    tables[0, :T] = idx
    tables[1, :T] = idx * idx + 3
    tables[2, :T] = idx ^ 0x5555
    tables[3, :T] = 1
    picks = wrnd((NSUB, n), T)
    lk_cols = torch.stack([tables[j][picks[i]] for i in range(NSUB) for j in range(W)])
    mult = torch.bincount(picks.reshape(-1), minlength=n).to(torch.int64)
    boolean = wrnd((1, n), 2)
    variables = torch.cat([gp, lk_cols, boolean], dim=0)
    # sigmas: identity k_j * omega^i, then the chained cells of fma / reduction rows swapped
    ks = ctx.non_residues_for_copy_permutation(n, V)
    mono = torch.zeros((V, n), dtype=torch.int64, device=dev)
    mono[:, 1 if n > 1 else 0] = torch.from_numpy(ks.view(np.int64)).to(dev)
    ctx.fft_natural_to_bitreversed(mono, 1)
    ctx.bitreverse_enumeration_inplace(mono)
    ident = mono
    sigmas = ident.clone()
    for k in range(1, n_fma):
        a, b = 4 * k + 2, 4 * k - 1
        sigmas[a] = torch.where(is_fma, ident[b], sigmas[a])
        sigmas[b] = torch.where(is_fma, ident[a], sigmas[b])
    for k in range(1, n_red):
        a, b = 5 * k, 5 * k - 1
        sigmas[a] = torch.where(is_red, ident[b], sigmas[a])
        sigmas[b] = torch.where(is_red, ident[a], sigmas[b])
    lk = dict(width=W, num_repetitions=NSUB, variables_offset=GP, table_id_column=7, tables=tables.contiguous(), multiplicities=mult.contiguous())
    pi_row = (n * 1041222) >> 20            # the fixture publishes row 1041222 of 2^20
    return dict(variables=variables.contiguous(), sigmas=sigmas.contiguous(), constants=constants.contiguous(), gates=gates,
                quotient_degree=8, lookup=lk, public_inputs=[(c, pi_row) for c in range(4)])
