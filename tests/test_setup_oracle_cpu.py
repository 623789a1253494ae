"""The C oracle of the setup's host loops (oracle/oracle.c: orc_create_permutation_polys, orc_materialize_columns) pinned to
their line-by-line Python restatement (oracle/setup_oracle.py) on many small random placements and on every edge case the GPU
tests of bj_create_permutation_polys / bj_materialize_columns use at production sizes; and the u32 conversion of the variables
copy hint (bj_variables_hint_to_u32) at the edges of its index range."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import setup_oracle as SO

P = O.P
PH = 1 << 63                  # Variable::placeholder
LOW48 = (1 << 48) - 1


def _lists(a):
    return [[int(v) for v in col] for col in a]


def _sigma_py(place):
    return np.array(SO.create_permutation_polys(_lists(place), place.shape[1]), dtype=np.uint64)


def _identity(n_cols, n):
    return _sigma_py(np.full((n_cols, n), PH, np.uint64))


def _random_placement(r, n_cols, n):
    """variables used 1..4 times at random cells, indices spread over the 48-bit range, 10 % placeholders"""
    cells = n_cols * n
    mult = r.integers(1, 5, size=cells)
    k = int(np.searchsorted(np.cumsum(mult), cells)) + 1
    ids = (np.arange(k, dtype=np.uint64) * np.uint64(0x9E3779B97F4B)) & np.uint64(LOW48)
    flat = np.repeat(ids, mult[:k])[:cells]
    flat = flat[r.permutation(cells)]
    flat[r.random(cells) < 0.1] = np.uint64(PH)
    return flat.reshape(n_cols, n)


def _edge_cases(n_cols, n):
    """(name, placement) of the cases the GPU tests also run at production sizes"""
    cells = n_cols * n
    r = np.random.default_rng(n_cols * 1000 + n)
    out = {}
    base = _random_placement(r, n_cols, n)
    one = base.copy()
    one[1] = 77                                                     # one variable fills a whole column
    out["one_variable_fills_a_column"] = one
    out["all_self_loops"] = np.arange(cells, dtype=np.uint64).reshape(n_cols, n) * np.uint64(3)
    out["all_placeholders"] = np.full((n_cols, n), PH, np.uint64)
    col = base.copy()
    col[n_cols - 1] = PH                                            # one column entirely placeholders
    out["one_column_of_placeholders"] = col
    ends = base.copy()
    ends[0, 0] = ends[-1, -1] = ends[n_cols // 2, n // 2] = 123456789   # the first and the last cell of the flat order in one group
    out["first_and_last_cell_in_one_group"] = ends
    hi = base.copy()
    v = np.uint64(0x5_0000_0007)
    vals = [LOW48, LOW48 - 1, 0, int(v), int(v) + (1 << 32), int(v) - (1 << 32), 7, (1 << 32) + 7]
    pos = r.choice(cells, size=4 * len(vals), replace=False)
    hi.reshape(-1)[pos] = np.repeat(np.array(vals, dtype=np.uint64), 4)   # indices equal in their low 32 bits, and at the ends
    out["indices_at_the_ends_and_equal_low_32_bits"] = hi
    junk = base.copy()
    f = junk.reshape(-1)
    live = (f & np.uint64(PH)) == 0
    f[live] |= r.integers(1, 1 << 15, size=int(live.sum()), dtype=np.uint64) << np.uint64(48)   # junk in bits 48..62
    out["junk_in_bits_48_to_62"] = junk
    lowph = base.copy()
    f = lowph.reshape(-1)
    ph = (f & np.uint64(PH)) != 0
    f[ph] |= r.integers(0, 1 << 63, size=int(ph.sum()), dtype=np.uint64)   # placeholders with any low bits
    out["placeholders_with_low_bits"] = lowph
    return out, base


@pytest.mark.parametrize("seed", range(24))
def test_sigma_c_oracle_equals_python_on_random_placements(seed):
    r = np.random.default_rng(seed)
    log_n, n_cols = int(r.integers(0, 8)), int(r.integers(1, 9))
    n = 1 << log_n
    n_vars = int(r.integers(1, 2 * n_cols * n + 2))
    place = (r.integers(0, n_vars, size=(n_cols, n), dtype=np.uint64) * np.uint64(seed + 1)) & np.uint64(LOW48)
    place[r.random((n_cols, n)) < 0.2] = np.uint64(PH)
    assert np.array_equal(O.create_permutation_polys(place), _sigma_py(place))


@pytest.mark.parametrize("log_n,n_cols", [(4, 3), (6, 5), (9, 4)])
def test_sigma_c_oracle_equals_python_on_the_edge_cases(log_n, n_cols):
    n = 1 << log_n
    cases, base = _edge_cases(n_cols, n)
    ident = _identity(n_cols, n)
    assert np.array_equal(O.create_permutation_polys(np.full((n_cols, n), PH, np.uint64)), ident)
    for name, place in cases.items():
        got = O.create_permutation_polys(place)
        assert np.array_equal(got, _sigma_py(place)), name
        assert np.array_equal(np.sort(got, axis=None), np.sort(ident, axis=None)), name
    assert np.array_equal(O.create_permutation_polys(cases["all_self_loops"]), ident)
    assert np.array_equal(O.create_permutation_polys(cases["junk_in_bits_48_to_62"]), O.create_permutation_polys(base))
    assert np.array_equal(O.create_permutation_polys(cases["placeholders_with_low_bits"]), O.create_permutation_polys(base))


def test_sigma_c_oracle_grows_its_scratch_table():
    """more distinct variables than the scratch table's first capacity (2^16): the table is rehashed on the way"""
    r = np.random.default_rng(5)
    place = _random_placement(r, 3, 1 << 16)
    got = O.create_permutation_polys(place)
    assert np.array_equal(got, _sigma_py(place))


def test_sigma_of_a_two_cycle_swaps_identity_values():
    n = 8
    place = np.full((2, n), PH, np.uint64)
    place[0, 3] = place[1, 5] = 9
    ident = _identity(2, n)
    want = ident.copy()
    want[0, 3], want[1, 5] = ident[1, 5], ident[0, 3]
    assert np.array_equal(O.create_permutation_polys(place), want)


def _lazy(r, values, frac=0.3):
    """values with p added to a seeded share of the ones below 2^32 - 1: non-canonical words of the same field elements"""
    v = values.copy()
    small = np.flatnonzero(v < np.uint64(2**32 - 1))
    v[small[r.random(small.size) < frac]] += np.uint64(P)
    return v


@pytest.mark.parametrize("seed", range(16))
def test_materialize_c_oracle_equals_python(seed):
    r = np.random.default_rng(100 + seed)
    log_n, n_cols = int(r.integers(0, 9)), int(r.integers(1, 7))
    n = 1 << log_n
    hint_rows = int(r.choice([n, max(n - 1, 1), 1, int(r.integers(1, n + 1))]))
    n_values = int(r.integers(1, 400))
    values = _lazy(r, O.random_field(r, n_values) >> r.integers(0, 40, size=n_values, dtype=np.uint64))
    values[: min(3, n_values)] = [P, P + 9, 2**64 - 1][: min(3, n_values)]
    hint = r.integers(0, n_values, size=(n_cols, hint_rows), dtype=np.uint64)
    hint[r.random((n_cols, hint_rows)) < 0.2] = np.uint64(PH)
    got, bad = O.materialize_columns(values, hint, log_n)
    assert bad == 0
    assert got.tolist() == SO.materialize_columns([int(v) for v in values], _lists(hint), n)


def test_materialize_c_oracle_masks_and_counts():
    values = np.array([5, P + 3, 2**64 - 1, 11], dtype=np.uint64)
    hint = np.array([[1, PH | 2, 2 | (0x7ABC << 48), 4, 0]], dtype=np.uint64)
    got, bad = O.materialize_columns(values, hint, 3)
    assert got.tolist() == [[3, 0, (2**64 - 1) % P, 0, 5, 0, 0, 0]] and bad == 1


# ---- bj_variables_hint_to_u32 at the edges of the u32 index range ----
@pytest.fixture(scope="module")
def bj():
    import era_boojum_b200 as m
    return m


def test_hint_u32_accepts_the_largest_index_and_masks_bits_48_to_62(bj):
    junk = np.uint64(0x7FFF << 48)
    h = np.array([[(1 << 32) - 2, 5 | (1 << 48), 9 | int(junk), PH, PH | 0x1234, PH | LOW48, 0]], dtype=np.uint64)
    out, need = bj.variables_hint_to_u32(h)
    assert out.tolist() == [[(1 << 32) - 2, 5, 9, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0]]
    assert need == (1 << 32) - 1


@pytest.mark.parametrize("word", [(1 << 32) - 1, ((1 << 32) - 1) | (0x55 << 48), (1 << 32) | (1 << 62)])
def test_hint_u32_refuses_the_placeholder_index(bj, word):
    h = np.array([[0, word]], dtype=np.uint64)
    with pytest.raises(bj.BoojumError) as e:
        bj.variables_hint_to_u32(h)
    assert e.value.status == bj.native.BJ_ERR_INVALID_ARG
