"""The C oracle of recorded gate programs (orc_gates_quotient / orc_gates_check in oracle/oracle.c) tied, without a GPU, to the
Python-int oracles it restates at small sizes: oracle/gates.py's quotient row, the gate library's own evaluators
(era_boojum_b200/gate_library.py, pinned by the quotient identity on the reference's proof.json) for all 11 gates incl. the
Poseidon2 flattened gate, a direct evaluation of programs that read witness columns, and oracle/satisfiability.py's gate report on
the mutation catalogue of tests/test_satisfiability_cpu.py.  Inputs include non-canonical values (x + p, 2^64 - 1).  The GPU
tests of the interpreter (tests/test_gpu_gate_interpreter.py) compare the device with this oracle over whole vectors."""
import random

import numpy as np
import pytest

from era_boojum_b200 import gate_library as GL
from era_boojum_b200 import native as N
from era_boojum_b200 import synthetic
from oracle import gates as OG
from oracle import oracle as O
from oracle import verifier_reference as VR
from tests import test_satisfiability_cpu as CAT

P = O.P
LIBRARY = [GL.CONSTANT_ALLOCATOR, GL.BOOLEAN, GL.FMA, GL.REDUCTION4, GL.DOT_PRODUCT4, GL.ZERO_CHECK, GL.UINTX_ADD, GL.SELECTION,
           GL.PARALLEL_SELECTION4, GL.U8X4_FMA, GL.poseidon2_flattened_gate(130, 0)]


def lazy_columns(rnd, n_cols, n):
    """[n_cols, n] u64 mixing canonical values, their non-canonical twins (x + p) and the edges 0, 1, p - 1, p, p + 1, 2^64 - 1"""
    edges = [0, 1, P - 1, P, P + 1, 2**64 - 1, 2**32, (1 << 32) - 1]
    out = np.zeros((n_cols, n), np.uint64)
    for c in range(n_cols):
        for t in range(n):
            x = rnd.random()
            v = rnd.choice(edges) if x < 0.2 else rnd.randrange(P)
            if 0.2 <= x < 0.4 and v < 2**64 - P:
                v += P
            out[c, t] = v
    return out


def alphas_for(rnd, n_terms):
    return [(rnd.randrange(2**64), rnd.randrange(2**64)) for _ in range(n_terms)]   # non-canonical powers too


def test_sha_layout_matches_the_quotient_row():
    """oracle/gates.py quotient_gates_row (the bench gates by name) at every point, q added to non-canonical initial values"""
    rnd = random.Random(1)
    n, V, C = 40, 60, 6
    gates = synthetic.sha_shaped_gates(V)
    layout = [(g["name"], g["num_repetitions"], g["selector_path"]) for g in gates]
    var, con = lazy_columns(rnd, V, n), lazy_columns(rnd, C, n)
    con[:2, : n // 2] = np.array([[rnd.choice([0, 1, P, P + 1]) for _ in range(n // 2)] for _ in range(2)], np.uint64)
    n_terms = sum(g["num_repetitions"] * len(g["writes"]) for g in gates)
    al = alphas_for(rnd, n_terms)
    q0, q1 = lazy_columns(rnd, 2, n)
    g0, g1 = O.gates_quotient(gates, var, [], con, al, q0, q1)
    alc = [(a % P, b % P) for a, b in al]
    for t in range(n):
        w0, w1 = OG.quotient_gates_row(layout, [int(x) % P for x in var[:, t]], [int(x) % P for x in con[:, t]], alc)
        assert (int(g0[t]), int(g1[t])) == ((int(q0[t]) + w0) % P, (int(q1[t]) + w1) % P), t


def test_production_layout_matches_the_quotient_row():
    """the production-shaped gate set (11 recorded programs, the Poseidon2 flattened gate among them, 415 terms) through
    quotient_gates_row's program path"""
    from tests.test_oracle_prover_cpu import production_gates
    dicts, tuples = production_gates()
    rnd = random.Random(2)
    n, V, C = 6, 155, 8
    var, con = lazy_columns(rnd, V, n), lazy_columns(rnd, C, n)
    al = alphas_for(rnd, 415)
    q0, q1 = lazy_columns(rnd, 2, n)
    g0, g1 = O.gates_quotient(dicts, var, [], con, al, q0, q1)
    alc = [(a % P, b % P) for a, b in al]
    for t in range(n):
        w0, w1 = OG.quotient_gates_row(tuples, [int(x) % P for x in var[:, t]], [int(x) % P for x in con[:, t]], alc)
        assert (int(g0[t]), int(g1[t])) == ((int(q0[t]) + w0) % P, (int(q1[t]) + w1) % P), t


def _library_case(gate, seed, n):
    rnd = random.Random(seed)
    reps = min(3, gate.num_repetitions_in_geometry(130, 0, 8))
    path = [rnd.random() < 0.5 for _ in range(rnd.randrange(0, 4))]
    var0 = rnd.randrange(0, 4)
    placed = GL.placed(gate, reps, path, variables_initial_offset=var0)
    V = var0 + max(130, gate.width[0] * reps)
    C = len(path) + max(gate.width[2] * reps, gate.shared, 1)
    var, con = lazy_columns(rnd, V, n), lazy_columns(rnd, C, n)
    for i in range(len(path)):                                # selector columns: mostly 0 / 1 (also as p, p + 1)
        con[i] = [rnd.choice([0, 1, P, P + 1, rnd.randrange(P)]) for _ in range(n)]
    return rnd, placed, reps, path, var0, var, con


def _library_terms(gate, reps, path, var0, var, con, t):
    vr, cr = [int(x) % P for x in var[:, t]], [int(x) % P for x in con[:, t]]
    terms = GL.evaluate_gate_terms(gate, VR.BaseBackend, lambda i: vr[i], lambda i: 0, lambda i: cr[i], reps, var_base=var0,
                                   const_base=len(path))
    return [int(x) % P for x in terms], OG.selector(path, cr)


@pytest.mark.parametrize("gate", LIBRARY, ids=lambda g: g.name)
def test_library_gates_quotient(gate):
    n = 4 if gate.name.startswith("poseidon2") else 12
    rnd, placed, reps, path, var0, var, con = _library_case(gate, LIBRARY.index(gate), n)
    al = alphas_for(rnd, reps * gate.terms)
    q0, q1 = lazy_columns(rnd, 2, n)
    g0, g1 = O.gates_quotient([placed], var, [], con, al, q0, q1)
    for t in range(n):
        terms, sel = _library_terms(gate, reps, path, var0, var, con, t)
        w0 = sum(x * a[0] for x, a in zip(terms, al)) * sel
        w1 = sum(x * a[1] for x, a in zip(terms, al)) * sel
        assert (int(g0[t]), int(g1[t])) == ((int(q0[t]) + w0) % P, (int(q1[t]) + w1) % P), t


@pytest.mark.parametrize("gate", LIBRARY, ids=lambda g: g.name)
def test_library_gates_check(gate):
    """check mode on random rows (most terms nonzero): per row the first failing (repetition, term), its value and selector;
    failures counted per (row, repetition) where the selector is nonzero"""
    n = 4 if gate.name.startswith("poseidon2") else 12
    rnd, placed, reps, path, var0, var, con = _library_case(gate, 100 + LIBRARY.index(gate), n)
    for t in range(0, n, 3):                                   # a few rows that satisfy the gate: all variables 0, constants 0
        var[:, t] = 0
        con[len(path):, t] = 0
    got = O.gates_check([placed], var, con)
    fails, first = 0, None
    for t in range(n):
        terms, sel = _library_terms(gate, reps, path, var0, var, con, t)
        fv = fs = 0
        if sel:
            for rep in range(reps):
                bad = [j for j in range(gate.terms) if terms[rep * gate.terms + j]]
                if bad:
                    fails += 1
                    if not fv:
                        fv, fs = terms[rep * gate.terms + bad[0]], sel
                        first = first or (t, rep * gate.terms + bad[0])
        assert (int(got["first_value"][t]), int(got["first_selector"][t])) == (fv, fs), t
    assert got["failures"] == fails
    assert (got["row"], got["term"]) == (first or (0, 0))


def test_witness_columns_and_strides():
    """operands of every column kind with per-repetition strides and initial offsets (witnesses too), immediates at and above
    p, INVERSE of 0 and of p, against a direct evaluation"""
    V_, W_, C_, CS, T, K = N.IDX_VARIABLE, N.IDX_WITNESS, N.IDX_CONSTANT_POLY, N.IDX_CONSTANT_POLY_SHARED, N.IDX_TEMPORARY, N.IDX_CONSTANT_VALUE
    rel = [(N.REL_MUL, 0, (W_, 1), (V_, 0)), (N.REL_ADD, 1, (T, 0), (CS, 1)), (N.REL_SUB, 2, (C_, 0), (W_, 0)),
           (N.REL_INVERSE, 3, (T, 2), None), (N.REL_MUL, 4, (T, 3), (K, 2**64 - 1)), (N.REL_SQUARE, 5, (V_, 1), None),
           (N.REL_NEGATE, 6, (T, 5), None), (N.REL_DOUBLE, 7, (W_, 1), None), (N.REL_INVERSE, 8, (K, P), None),
           (N.REL_ADD, 9, (T, 8), (T, 7))]
    gate = dict(relations=rel, writes=[(T, 1), (T, 4), (T, 6), (W_, 1), (T, 9), (K, P + 5)], num_repetitions=3, variables_offset=2,
                witnesses_offset=3, constants_offset=1, constants_placement_offset=2, selector_path=[True, False],
                variables_initial_offset=1, witnesses_initial_offset=2)
    rnd = random.Random(3)
    n, V, W, C = 24, 8, 12, 6
    var, wit, con = lazy_columns(rnd, V, n), lazy_columns(rnd, W, n), lazy_columns(rnd, C, n)
    wit[2, ::4] = 0
    wit[2, 1::4] = P
    con[2, ::4] = 0                                            # C_ 0 - W_ 0 = 0 on every fourth row of repetition 0: INVERSE(0)
    al = alphas_for(rnd, 18)
    q0, q1 = lazy_columns(rnd, 2, n)
    g0, g1 = O.gates_quotient([gate], var, wit, con, al, q0, q1)
    for t in range(n):
        v, w, c = ([int(x) % P for x in a[:, t]] for a in (var, wit, con))
        terms = []
        for rep in range(3):
            vb, wb, cb = 1 + 2 * rep, 2 + 3 * rep, 2 + rep
            t0 = w[wb + 1] * v[vb]
            t2 = (c[cb] - w[wb]) % P
            t3 = pow(t2, P - 2, P)
            terms += [(t0 + c[2 + 1]) % P, t3 * ((2**64 - 1) % P) % P, (-v[vb + 1] ** 2) % P, w[wb + 1], 2 * w[wb + 1] % P, 5]
        sel = c[0] * (1 - c[1]) % P
        w0 = sum(x * (a[0] % P) for x, a in zip(terms, al)) * sel
        w1 = sum(x * (a[1] % P) for x, a in zip(terms, al)) * sel
        assert (int(g0[t]), int(g1[t])) == ((int(q0[t]) + w0) % P, (int(q1[t]) + w1) % P), t
    assert all(int(x) < P for x in np.concatenate([g0, g1]))


def _gate_fields(report):
    return {k: v for k, v in report.items() if k.startswith("gate_")}


@pytest.mark.parametrize("mutation", CAT.SHA_MUTATIONS, ids=lambda m: m.__name__)
def test_mutation_catalogue_sha(mutation):
    m, want = CAT.mutated(CAT.sha_circuit(6), mutation)
    got = O.gates_report(m["gates"], m["variables"], m["constants"])
    assert got == _gate_fields(CAT.oracle_report(m)) == _gate_fields(want)


@pytest.mark.parametrize("mutation", CAT.PRODUCTION_MUTATIONS, ids=lambda m: m.__name__)
def test_mutation_catalogue_production(mutation):
    m, want = CAT.mutated(CAT.production_circuit(5), mutation)
    got = O.gates_report(m["gates"], m["variables"], m["constants"])
    assert got == _gate_fields(CAT.oracle_report(m)) == _gate_fields(want)


def test_satisfied_circuits_report_nothing():
    for c in (CAT.sha_circuit(7), CAT.production_circuit(5)):
        assert O.gates_report(c["gates"], c["variables"], c["constants"])["gate_failures"] == 0
