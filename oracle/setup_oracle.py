"""TEST ORACLE (never imported by the product): Python restatement of the reference's host loops that build the witness
columns and the sigma columns.  Follows the reference line by line; small sizes only (oracle.c's orc_materialize_columns and
orc_create_permutation_polys restate the same loops for production sizes and are pinned to these by
tests/test_setup_oracle_cpu.py).

  materialize_variables_polynomials_from_dense_hint   src/cs/implementations/witness.rs:325-385
  create_permutation_polys                            src/cs/implementations/setup.rs:419-502
  Variable encoding                                    src/cs/mod.rs:44-47, :155-180
"""
from .replay import P, omega
from .stage2 import non_residues_for_copy_permutation as non_residues

PLACEHOLDER_BIT = 1 << 63
LOW_U48 = (1 << 48) - 1


def materialize_columns(all_values, hint, n):
    """hint: list of columns, each a list of Variables (ints).  witness.rs:363-381."""
    out = []
    for col in hint:
        poly = [0] * n
        for row, var in enumerate(col):
            if not (var & PLACEHOLDER_BIT):
                poly[row] = all_values[var] % P
        out.append(poly)
    return out


def create_permutation_polys(placement, n):
    """placement: copy_permutation_data, list of columns of Variables.  setup.rs:436-489."""
    log_n = n.bit_length() - 1
    w = omega(log_n)
    nrs = non_residues(n, len(placement))
    result = []
    for k in nrs:                                  # materialize_x_by_non_residue_polys
        x, col = 1, []
        for _ in range(n):
            col.append(k * x % P)
            x = x * w % P
        result.append(col)
    scratch = {}                                    # var index -> [stored value, (first column, first row)]
    for column_idx, column in enumerate(placement):
        poly = result[column_idx]
        for row, var in enumerate(column):
            if var & PLACEHOLDER_BIT:
                continue
            var_idx = var & LOW_U48
            if var_idx not in scratch:
                scratch[var_idx] = [poly[row], (column_idx, row)]
            else:                                   # std::mem::swap(&mut previous.0, &mut poly.storage[row])
                scratch[var_idx][0], poly[row] = poly[row], scratch[var_idx][0]
    for value, (c, r) in scratch.values():          # close the cycles: the last occurrence goes to the first
        result[c][r] = value
    return result
