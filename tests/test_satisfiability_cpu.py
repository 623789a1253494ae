"""The satisfiability check without a GPU: the oracle's restatement (oracle/satisfiability.py) reports nothing on the generated
circuits and, on a catalogue of mutations, exactly the report written down from each mutation's construction.  The same
catalogue drives the device check in tests/test_gpu_satisfiability.py.  Also: the sigma decode is well defined (the k_c^n are
pairwise distinct) and the report struct has the same size in ctypes and in C."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import circuits
from oracle import satisfiability as OS
from oracle.gates import P
from oracle.replay import omega
from oracle.stage2 import non_residues_for_copy_permutation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V_SHA = 20   # general-purpose columns of the SHA-shaped mutation circuits (5 FMA repetitions, 4 reduction repetitions)


def sha_circuit(log_n, seed=7, V=V_SHA, lookup=True):
    """circuits.sha_shaped with its gates as the library takes them (recorded programs) and as the oracle takes them"""
    from era_boojum_b200 import synthetic
    c = circuits.sha_shaped(log_n, V, seed=seed, lookup=lookup)
    c["oracle_gates"] = c["gates"]
    c["gates"] = synthetic.sha_shaped_gates(V)
    assert [(g["name"], g["num_repetitions"], g["selector_path"]) for g in c["gates"]] == [tuple(g) for g in c["oracle_gates"]]
    return c


def production_circuit(log_n, seed=3):
    from tests.test_oracle_prover_cpu import production_gates
    c = circuits.production_shaped(log_n, seed=seed)
    dicts, tuples = production_gates()
    c["gates"], c["oracle_gates"] = dicts, tuples
    return c


def copy_circuit(c):
    out = dict(c, variables=c["variables"].copy(), sigmas=c["sigmas"].copy(), constants=c["constants"].copy())
    if c["lookup"]:
        out["lookup"] = dict(c["lookup"], tables=c["lookup"]["tables"].copy(), multiplicities=c["lookup"]["multiplicities"].copy())
    return out


def expect(**fields):
    r = OS.empty_report()
    r.update(fields)
    return OS.finish(r)


def oracle_report(c):
    return OS.check(c["variables"], c["sigmas"], c["constants"], c["oracle_gates"], c["lookup"])


# ---- row kinds of circuits.sha_shaped (selector columns 0, 1) ----
def sha_rows(c, kind):
    con = c["constants"]
    sel = {"ca": (con[0] == 1) & (con[1] == 1), "fma": (con[0] == 1) & (con[1] == 0), "red": con[0] == 0}[kind]
    return [int(r) for r in np.nonzero(sel)[0]]


def _pick(rows, which):
    return rows[0] if which == "first" else rows[-1]


# ---- the mutation catalogue: each mutates a copy of the circuit in place and returns the report it must produce ----
def fma_output(c, which="last"):
    """the output d of the last FMA repetition (column 19, tied to nothing) + 1: that repetition's term is -1"""
    r = _pick(sha_rows(c, "fma"), which)
    c["variables"][19, r] = (int(c["variables"][19, r]) + 1) % P
    return expect(gate_failures=1, gate_row=r, gate_index=1, gate_repetition=4, gate_term=0, gate_value=P - 1, gate_selector=1)


def reduction_output(c, which="last"):
    """the output of the last reduction repetition (column 19) + 1"""
    r = _pick(sha_rows(c, "red"), which)
    c["variables"][19, r] = (int(c["variables"][19, r]) + 1) % P
    return expect(gate_failures=1, gate_row=r, gate_index=2, gate_repetition=3, gate_term=0, gate_value=P - 1, gate_selector=1)


def _fma_terms(c, r):
    v, con = [int(x) for x in c["variables"][:, r]], [int(x) for x in c["constants"][:, r]]
    return [(con[2] * v[4 * k] * v[4 * k + 1] + con[3] * v[4 * k + 2] - v[4 * k + 3]) % P for k in range(V_SHA // 4)]


def selector_flip(c, which="last"):
    """constant column 1 of a constants-allocator row set to 0: the row now selects the FMA gate, whose 5 repetitions all fail"""
    rows = [r for r in sha_rows(c, "ca")]
    r = _pick(rows, which)
    c["constants"][1, r] = 0
    terms = _fma_terms(c, r)
    assert all(terms)
    return expect(gate_failures=len(terms), gate_row=r, gate_index=1, gate_repetition=0, gate_term=0, gate_value=terms[0], gate_selector=1)


def constant_change(c, which="last"):
    """the quadratic coefficient of an FMA row + 1: every repetition's term becomes a_k * b_k"""
    v = c["variables"]
    rows = [r for r in sha_rows(c, "fma") if all(int(v[4 * k, r]) * int(v[4 * k + 1, r]) % P for k in range(V_SHA // 4))]
    r = _pick(rows, which)
    c["constants"][2, r] += 1
    return expect(gate_failures=V_SHA // 4, gate_row=r, gate_index=1, gate_repetition=0, gate_term=0,
                  gate_value=int(v[0, r]) * int(v[1, r]) % P, gate_selector=1)


def tied_pair(c, which="last"):
    """input c of FMA repetition 1 (column 6, tied to the output of repetition 0 in column 3) + 1: two copy failures, and
    repetition 1's term becomes its linear coefficient"""
    rows = [r for r in sha_rows(c, "fma") if int(c["constants"][3, r])]
    r = _pick(rows, which)
    v = c["variables"]
    v[6, r] = (int(v[6, r]) + 1) % P
    return expect(copy_failures=2, copy_row=r, copy_column=3, copy_other_row=r, copy_other_column=6, copy_value=int(v[3, r]),
                  copy_other_value=int(v[6, r]), gate_failures=1, gate_row=r, gate_index=1, gate_repetition=1, gate_term=0,
                  gate_value=int(c["constants"][3, r]), gate_selector=1)


def sigma_swap(c, which="last"):
    """the sigma entries of cells (column 0, row 1) and (column 1, row n - 1), never tied, swapped: each names the other"""
    n = c["variables"].shape[1]
    r1, r2 = 1, n - 1
    s, v = c["sigmas"], c["variables"]
    assert int(v[0, r1]) != int(v[1, r2])
    s[0, r1], s[1, r2] = int(s[1, r2]), int(s[0, r1])
    return expect(copy_failures=2, copy_row=r1, copy_column=0, copy_other_row=r2, copy_other_column=1, copy_value=int(v[0, r1]),
                  copy_other_value=int(v[1, r2]))


def sigma_non_coset(c, which="last"):
    """the sigma entry of cell (column 2, row n - 1) replaced by k_V w^row, k_V the next non-residue (no column has it): that
    entry names no cell, and its cell is named by no entry"""
    V, n = c["variables"].shape
    r = n - 1
    k = non_residues_for_copy_permutation(n, V + 1)[V]
    c["sigmas"][2, r] = k * pow(omega(n.bit_length() - 1), r, P) % P
    return expect(sigma_failures=2, sigma_row=r, sigma_column=2, sigma_kind=OS.SIGMA_NO_CELL)


def lookup_off_table(c, which="last"):
    """the first lookup column of sub-argument 0 on row n - 1 set to p - 1 (in no table row): one unmatched tuple, and the
    table row it matched before is counted once less than its multiplicity"""
    lk = c["lookup"]
    n = c["variables"].shape[1]
    r, col = n - 1, lk["variables_offset"]
    pick = int(c["variables"][col, r])            # table column 0 holds the row index
    c["variables"][col, r] = P - 1
    m = int(lk["multiplicities"][pick])
    return expect(lookup_unmatched=1, lookup_row=r, lookup_subargument=0, multiplicity_failures=1, multiplicity_row=pick,
                  multiplicity_count=m - 1, multiplicity_sum=m)


def multiplicity_plus(c, which="last", row=None):
    lk = c["lookup"]
    f = row if row is not None else min(c["variables"].shape[1], 1 << 10) - 1
    m = int(lk["multiplicities"][f])
    lk["multiplicities"][f] = m + 1
    return expect(multiplicity_failures=1, multiplicity_row=f, multiplicity_count=m, multiplicity_sum=m + 1)


def multiplicity_minus(c, which="last", row=0):
    lk = c["lookup"]
    m = int(lk["multiplicities"][row])
    lk["multiplicities"][row] = (m - 1) % P
    return expect(multiplicity_failures=1, multiplicity_row=row, multiplicity_count=m, multiplicity_sum=(m - 1) % P)


def padding_multiplicity(c, which="last"):
    """a multiplicity of 1 on a padding row (table rows T..n-1 are all zero, T = 2^10): the zero content, first found at row T,
    is looked up by no tuple"""
    T = 1 << 10
    assert c["variables"].shape[1] > T
    c["lookup"]["multiplicities"][T + 5] = 1
    return expect(multiplicity_failures=1, multiplicity_row=T, multiplicity_count=0, multiplicity_sum=1)


_KEYS = {"gate": ("gate_row", "gate_index", "gate_repetition", "gate_term"), "copy": ("copy_row", "copy_column"),
         "sigma": ("sigma_row", "sigma_column", "sigma_kind"), "lookup": ("lookup_row", "lookup_subargument"),
         "multiplicity": ("multiplicity_row",)}
_COUNTS = {"gate": "gate_failures", "copy": "copy_failures", "sigma": "sigma_failures", "lookup": "lookup_unmatched",
           "multiplicity": "multiplicity_failures"}


def merge(reports):
    """the report of independent failures: counts add, each kind's first is the one with the smallest key"""
    out = OS.empty_report()
    for kind, cnt in _COUNTS.items():
        having = [r for r in reports if r[cnt]]
        if not having:
            continue
        best = min(having, key=lambda r: tuple(r[k] for k in _KEYS[kind]))
        for f in OS.REPORT_FIELDS:
            if f.startswith(kind + "_") or f == cnt:
                out[f] = best[f]
        out[cnt] = sum(r[cnt] for r in having)
    return OS.finish(out)


def several(c, which="last"):
    """six failures at once, chosen so that the first of each kind is not the last one applied"""
    return merge([reduction_output(c, "last"), constant_change(c, "first"), sigma_swap(c), sigma_non_coset(c),
                  multiplicity_plus(c), multiplicity_minus(c)])


def production_boolean(c, which="last"):
    """the boolean gate's specialised column set to 2 on row n - 1: its term x - x^2 = -2 (no selector: the gate runs on every
    row)"""
    r = c["variables"].shape[1] - 1
    c["variables"][154, r] = 2
    return expect(gate_failures=1, gate_row=r, gate_index=0, gate_repetition=0, gate_term=0, gate_value=P - 2, gate_selector=1)


def production_fma_output(c, which="last"):
    """the output of the last FMA repetition (column 127) of the production shape's last FMA row + 1"""
    con = c["constants"]
    rows = [int(r) for r in np.nonzero((con[0] == 0) & (con[1] == 1) & (con[2] == 1) & (con[3] == 1) & (con[4] == 1))[0]]
    r = _pick(rows, which)
    c["variables"][127, r] = (int(c["variables"][127, r]) + 1) % P
    gi = [g["name"] for g in c["gates"]].index("fma")
    return expect(gate_failures=1, gate_row=r, gate_index=gi, gate_repetition=31, gate_term=0, gate_value=P - 1, gate_selector=1)


SHA_MUTATIONS = [fma_output, reduction_output, selector_flip, constant_change, tied_pair, sigma_swap, sigma_non_coset,
                 lookup_off_table, multiplicity_plus, multiplicity_minus, several]
PRODUCTION_MUTATIONS = [production_boolean, production_fma_output]


def mutated(c, mutation):
    m = copy_circuit(c)
    want = mutation(m)
    return m, want


# ---- tests ----
@pytest.mark.parametrize("log_n,V,lookup", [(5, 20, False), (6, 40, True), (7, 20, True), (8, 40, False)])
def test_oracle_reports_nothing_on_sha_shaped(log_n, V, lookup):
    c = sha_circuit(log_n, seed=log_n, V=V, lookup=lookup)
    assert oracle_report(c) == expect()


@pytest.mark.parametrize("log_n", [5, 6])
def test_oracle_reports_nothing_on_production_shaped(log_n):
    assert oracle_report(production_circuit(log_n, seed=log_n)) == expect()


@pytest.mark.parametrize("mutation", SHA_MUTATIONS, ids=lambda m: m.__name__)
def test_oracle_mutation_catalogue_sha(mutation):
    m, want = mutated(sha_circuit(6), mutation)
    assert want["satisfied"] == 0
    assert oracle_report(m) == want


@pytest.mark.parametrize("mutation", PRODUCTION_MUTATIONS, ids=lambda m: m.__name__)
def test_oracle_mutation_catalogue_production(mutation):
    m, want = mutated(production_circuit(5), mutation)
    assert oracle_report(m) == want


def test_oracle_padding_multiplicity():
    c = sha_circuit(11, V=20)
    m, want = mutated(c, padding_multiplicity)
    assert oracle_report(m) == want


def test_oracle_multiplicities_equal_the_circuit_column():
    c = sha_circuit(11, V=20)
    lk = c["lookup"]
    assert OS.multiplicities(c["variables"], c["constants"], lk) == [int(x) for x in lk["multiplicities"]]
    m, _ = mutated(c, lookup_off_table)
    assert OS.multiplicities(m["variables"], m["constants"], m["lookup"]) is None


def test_non_residue_powers_are_distinct():
    """the device decodes the column of a sigma entry s from s^n: for log_n <= 24 and V <= 256 the k_c^n of
    bj_non_residues_for_copy_permutation are pairwise distinct and, but for k_0 = 1, different from 1"""
    from era_boojum_b200 import native
    V = 256
    for log_n in range(1, 25):
        n = 1 << log_n
        out = (ctypes.c_uint64 * V)()
        assert native.lib.bj_non_residues_for_copy_permutation(n, V, out) == 0
        ks = [int(x) for x in out]
        assert ks == non_residues_for_copy_permutation(n, V)
        pw = [pow(k, n, P) for k in ks]
        assert pw[0] == 1 and all(x != 1 for x in pw[1:]) and len(set(pw)) == V


def test_report_struct_size_matches_c(tmp_path):
    from era_boojum_b200 import native
    src = tmp_path / "size.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "boojum_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", sizeof(bj_satisfiability_report), '
                   'offsetof(bj_satisfiability_report, sigma_kind), offsetof(bj_satisfiability_report, multiplicity_sum)); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.check_call(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, kind_off, sum_off = (int(x) for x in subprocess.check_output([str(exe)]).split())
    R = native.SatisfiabilityReport
    assert (size, kind_off, sum_off) == (ctypes.sizeof(R), R.sigma_kind.offset, R.multiplicity_sum.offset)
