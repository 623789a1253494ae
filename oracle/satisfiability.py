"""ORACLE (test infrastructure): the satisfiability check of a witness against its circuit, restated with Python ints and dicts
(small cases only) - the CPU counterpart of bj_check_satisfied, written independently of the device route.

  CSReferenceAssembly::check_if_satisfied          src/cs/implementations/satisfiability_test.rs:15-353
  materialize_multiplicities_polynomials           src/cs/implementations/witness.rs:225-272

Gates are evaluated with oracle/gates.py on the rows where their selector is nonzero; sigma entries are decoded with a plain
dict {k_c * w^r: (c, r)}; lookup tuples are matched with a dict {table row content: first row}.  check() returns the report in
the shape of bj_satisfiability_report (Context.check_if_satisfied): every count, and for each kind of failure the first one;
a "first" field is 0 when its count is 0.
"""
from .gates import GATES, P, program_terms, selector
from .replay import omega
from .stage2 import non_residues_for_copy_permutation

SIGMA_NO_CELL, SIGMA_UNNAMED, SIGMA_NAMED_TWICE = 1, 2, 3

REPORT_FIELDS = ("satisfied", "gate_failures", "gate_row", "gate_index", "gate_repetition", "gate_term", "gate_value", "gate_selector",
                 "copy_failures", "copy_row", "copy_other_row", "copy_column", "copy_other_column", "copy_value", "copy_other_value",
                 "sigma_failures", "sigma_row", "sigma_column", "sigma_kind", "lookup_unmatched", "lookup_row", "lookup_subargument",
                 "multiplicity_failures", "multiplicity_row", "multiplicity_count", "multiplicity_sum")


def empty_report():
    r = dict.fromkeys(REPORT_FIELDS, 0)
    r["satisfied"] = 1
    return r


def finish(r):
    """satisfied = no count is nonzero"""
    r["satisfied"] = int(not any(r[k] for k in ("gate_failures", "copy_failures", "sigma_failures", "lookup_unmatched",
                                                 "multiplicity_failures")))
    return r


def gate_terms(g, rep, var_row, const_row):
    """the terms of repetition `rep` of gate g = (name, reps, path[, first variable column, first constant column[, program]]),
    placed as oracle/gates.py quotient_gates_row places it"""
    name, path = g[0], g[2]
    var0 = g[3] if len(g) > 3 else 0
    place = g[4] if len(g) > 4 else len(path)
    if len(g) > 5:
        prog = g[5]
        return program_terms(prog, var_row, const_row, var0 + rep * prog["variables_offset"], place, place + rep * prog["constants_offset"])
    fn, width, _, (voff, coff) = GATES[name]
    return fn(var_row[var0 + rep * voff: var0 + rep * voff + width], const_row[place + rep * coff:])


def check_gates(variables, constants, gates, r):
    n = variables.shape[1]
    for row in range(n):
        var_row = [int(x) % P for x in variables[:, row]]
        const_row = [int(x) % P for x in constants[:, row]]
        for gi, g in enumerate(gates):
            sel = selector(g[2], const_row)
            if sel == 0:
                continue
            for rep in range(g[1]):
                bad = [(t, v % P) for t, v in enumerate(gate_terms(g, rep, var_row, const_row)) if v % P]
                if not bad:
                    continue
                if r["gate_failures"] == 0:
                    r.update(gate_row=row, gate_index=gi, gate_repetition=rep, gate_term=bad[0][0], gate_value=bad[0][1], gate_selector=sel)
                r["gate_failures"] += 1


def check_copy(variables, sigmas, r):
    V, n = variables.shape
    ks = non_residues_for_copy_permutation(n, V)
    w = omega(n.bit_length() - 1)
    cell_of = {}
    for c in range(V):
        x = ks[c]
        for row in range(n):
            cell_of[x] = (c, row)
            x = x * w % P
    named = {}
    sigma_bad = []                       # (row, column, kind)
    for row in range(n):
        for c in range(V):
            target = cell_of.get(int(sigmas[c, row]) % P)
            if target is None:
                sigma_bad.append((row, c, SIGMA_NO_CELL))
                continue
            named[target] = named.get(target, 0) + 1
            c2, r2 = target
            v, v2 = int(variables[c, row]) % P, int(variables[c2, r2]) % P
            if v != v2:
                if r["copy_failures"] == 0:
                    r.update(copy_row=row, copy_column=c, copy_other_row=r2, copy_other_column=c2, copy_value=v, copy_other_value=v2)
                r["copy_failures"] += 1
    for row in range(n):
        for c in range(V):
            k = named.get((c, row), 0)
            if k != 1:
                sigma_bad.append((row, c, SIGMA_UNNAMED if k == 0 else SIGMA_NAMED_TWICE))
    if sigma_bad:
        row, c, kind = min(sigma_bad)
        r.update(sigma_failures=len(sigma_bad), sigma_row=row, sigma_column=c, sigma_kind=kind)


def table_first_rows(tables):
    """{content: first row} over the rows of the table columns [width + 1, n] (table id last)"""
    first = {}
    for row in range(tables.shape[1]):
        first.setdefault(tuple(int(x) % P for x in tables[:, row]), row)
    return first


def lookup_counts(variables, constants, lookup):
    """-> ({first row: tuples equal to its content}, [(row, sub-argument) of the tuples that match no table row])"""
    W, R, voff, idc = lookup["width"], lookup["num_repetitions"], lookup["variables_offset"], lookup["table_id_column"]
    first = table_first_rows(lookup["tables"])
    count, unmatched = {}, []
    for row in range(variables.shape[1]):
        for i in range(R):
            t = tuple(int(variables[voff + i * W + j, row]) % P for j in range(W)) + (int(constants[idc, row]) % P,)
            f = first.get(t)
            if f is None:
                unmatched.append((row, i))
            else:
                count[f] = count.get(f, 0) + 1
    return count, unmatched


def check_lookup(variables, constants, lookup, r):
    count, unmatched = lookup_counts(variables, constants, lookup)
    if unmatched:
        r.update(lookup_unmatched=len(unmatched), lookup_row=unmatched[0][0], lookup_subargument=unmatched[0][1])
    tables, mult = lookup["tables"], lookup["multiplicities"]
    first = table_first_rows(tables)
    msum = {}
    for row in range(tables.shape[1]):
        f = first[tuple(int(x) % P for x in tables[:, row])]
        msum[f] = (msum.get(f, 0) + int(mult[row])) % P
    bad = sorted(f for f in set(first.values()) if count.get(f, 0) != msum.get(f, 0))
    if bad:
        f = bad[0]
        r.update(multiplicity_failures=len(bad), multiplicity_row=f, multiplicity_count=count.get(f, 0), multiplicity_sum=msum.get(f, 0))


def check(variables, sigmas, constants, gates, lookup=None):
    """the report of bj_check_satisfied.  variables / sigmas [V, n], constants [C, n] (numpy uint64); gates as oracle/gates.py
    takes them; lookup: dict(width, num_repetitions, variables_offset, table_id_column, tables [width + 1, n], multiplicities [n])"""
    r = empty_report()
    check_gates(variables, constants, gates, r)
    check_copy(variables, sigmas, r)
    if lookup:
        check_lookup(variables, constants, lookup, r)
    return finish(r)


def multiplicities(variables, constants, lookup):
    """materialize_multiplicities_polynomials: per table row, the number of tuples equal to its content if it is the content's
    first row, else 0 (None if a tuple matches no table row)"""
    count, unmatched = lookup_counts(variables, constants, lookup)
    if unmatched:
        return None
    out = [0] * lookup["tables"].shape[1]
    for f, k in count.items():
        out[f] = k
    return out
