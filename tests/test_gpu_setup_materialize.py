"""GPU tests of the setup's first steps at production sizes against the C oracle (oracle/oracle.c, pinned to the Python
restatement oracle/setup_oracle.py by tests/test_setup_oracle_cpu.py), every output compared over the whole array, bit for bit:
  - bj_create_permutation_polys (a radix sort of the cells by variable, a max-scan of group starts, a link kernel) on 155
    columns of 2^16, 2^20 and 2^21 rows, and on the placements where a sort or a scan goes wrong: a group longer than any
    sort tile or scan block, all self-loops, all or one column of placeholders, a group holding the first and the last cell,
    indices at the ends of the 48-bit range and pairs equal in their low 32 bits, junk in bits 48..62;
  - bj_materialize_columns and the u32 gather of bj_witness_upload_vec on 2^20 x 155 with non-canonical values;
  - the setup cap of bj_setup_create on the production geometry (LDE factor 2, quotient degree 8, cap 32, 155 sigma + 8
    constant + 4 table columns) on the resident, streamed and recompute plans, and of the compact plan (LDE factor 8,
    quotient degree 4), Poseidon2 and Blake2s, with the sigma columns coming from bj_create_permutation_polys: the chain
    placement -> sigma -> setup -> cap that a caller runs to get the verification key.
The verifier takes the setup cap as given, so a sigma that is a valid permutation but not the reference's would still give
proofs that verify; only a comparison with the reference's loops can see it."""
import hashlib

import numpy as np
import pytest

from oracle import oracle as O
from oracle import replay as R

pytestmark = pytest.mark.gpu

P = O.P
PH = 1 << 63                  # Variable::placeholder
LOW48 = (1 << 48) - 1
V = 155                       # columns under the copy permutation of the production geometry
SPREAD = 0x9E3779B97F4B       # odd: i -> i * SPREAD mod 2^48 is a bijection, so variable indices cover the 48-bit range
N20 = 1 << 20


@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import era_boojum_b200 as m
    return m


@pytest.fixture(scope="module")
def ctx(bj):
    c = bj.Context.on_current_stream(0)
    yield c
    c.synchronize()
    c.close()


_IDENT = {}
_SIGMA = {}
_PRODUCTION = {}
_CAPS = {}


@pytest.fixture(scope="module", autouse=True)
def release_caches():
    """the host arrays this module keeps between tests (up to a few GB) and the device blocks torch's allocator keeps after
    them are given back when the module ends, so later test modules see the memory they would see without it"""
    yield
    import gc
    import torch
    for cache in (_IDENT, _SIGMA, _PRODUCTION, _CAPS):
        cache.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _first_difference(got, want):
    diff = np.flatnonzero(got.reshape(-1) != want.reshape(-1))
    return "%d cells differ, first at flat cell %d" % (diff.size, diff[0]) if diff.size else ""


def placement(seed, log_n, n_cols=V, spread=True, placeholders=0.08):
    """a production-like copy_permutation_data [n_cols, 2^log_n]: variables used 1..4 times; the occurrences of one variable
    sit in neighbouring columns of a row (the row-major walk below), and 1 % of the cells trade places at random, so cycles cross
    columns and rows; a share of placeholder cells.  spread: indices over the whole 48-bit range, else 0, 1, 2, ..."""
    r = np.random.default_rng(seed)
    n = 1 << log_n
    cells = n_cols * n
    mult = r.integers(1, 5, size=cells // 2 + 16, dtype=np.int64)
    k = int(np.searchsorted(np.cumsum(mult), cells)) + 1
    ids = np.arange(k, dtype=np.uint64)
    if spread:
        ids = (ids * np.uint64(SPREAD)) & np.uint64(LOW48)
    place = np.ascontiguousarray(np.repeat(ids, mult[:k])[:cells].reshape(n, n_cols).T)
    f = place.reshape(-1)
    pick = r.integers(0, cells, size=cells // 100)
    f[pick] = f[r.permutation(pick)]
    f[r.integers(0, cells, size=int(cells * placeholders))] = np.uint64(PH)
    return place


def sorted_identity(n_cols, n):
    """the identity values k_c * w^row of every cell, sorted (a sigma is a permutation of them)"""
    if (n_cols, n) not in _IDENT:
        _IDENT[(n_cols, n)] = np.sort(O.create_permutation_polys(np.full((n_cols, n), PH, np.uint64)), axis=None)
    return _IDENT[(n_cols, n)]


def production_sigma(log_n):
    """(placement, the oracle's sigma) of the production-like placement at 2^log_n rows; kept up to 2^20 rows, where the setup
    tests take their sigma columns from it"""
    if log_n in _SIGMA:
        return _SIGMA[log_n]
    place = placement(log_n, log_n)
    out = (place, O.create_permutation_polys(place))
    if log_n <= 20:
        _SIGMA[log_n] = out
    return out


def check_sigma(bj, ctx, place, want=None):
    """GPU sigma == the oracle's over the whole array, and up to 2^20 rows also a permutation of the identity values (above
    that the sort costs more than it adds: the oracle's sigma is a permutation by construction) -> the sigma columns"""
    import torch
    got = bj.to_numpy(ctx.create_permutation_polys(bj.to_device(place)))
    torch.cuda.empty_cache()
    if want is None:
        want = O.create_permutation_polys(place)
    assert not _first_difference(got, want), _first_difference(got, want)
    if place.shape[1] <= N20:
        assert np.array_equal(np.sort(got, axis=None), sorted_identity(*place.shape))
    return got


# ------------------------------------------------------------------------------------------------------------ sigma -----
@pytest.mark.parametrize("log_n", [16, 20, 21])
def test_sigma_production_like(bj, ctx, log_n):
    """2^21 x 155 = 3.3e8 cells: the sort's tiles, the scan's multi-block carry and long groups all take part"""
    check_sigma(bj, ctx, *production_sigma(log_n))


def _edge_case(name, log_n=16):
    n = 1 << log_n
    cells = V * n
    r = np.random.default_rng(7)
    if name == "all_self_loops":
        return np.arange(cells, dtype=np.uint64).reshape(V, n) * np.uint64(3)
    if name == "all_placeholders":
        return np.full((V, n), PH, np.uint64)
    place = placement(1, log_n)
    if name == "one_variable_fills_a_column":
        place[40] = 12345           # 2^16 occurrences in one group: longer than a sort tile or a scan block
        place[41, ::97] = 12345
    elif name == "one_column_of_placeholders":
        place[V - 1] = PH
    elif name == "first_and_last_cell_in_one_group":
        place[0, 0] = place[V - 1, n - 1] = place[V // 2, n // 2] = 0x7777
    elif name == "indices_at_the_ends_and_equal_low_32_bits":
        # small indices elsewhere, so v and v + 2^32 sort next to each other with no index between them
        place = placement(2, log_n, spread=False)
        v = (1 << 33) + 5
        vals = [LOW48, LOW48 - 1, 0, v, v + (1 << 32), v + (2 << 32), 1 << 40, (1 << 40) + (1 << 32), LOW48 - (1 << 32)]
        pos = r.choice(cells, size=5 * len(vals), replace=False)
        place.reshape(-1)[pos] = np.repeat(np.array(vals, dtype=np.uint64), 5)
    elif name == "junk_in_bits_48_to_62":
        f = place.reshape(-1)
        live = (f & np.uint64(PH)) == 0
        f[live] |= r.integers(1, 1 << 15, size=int(live.sum()), dtype=np.uint64) << np.uint64(48)
    elif name == "placeholders_with_low_bits":
        f = place.reshape(-1)
        ph = (f & np.uint64(PH)) != 0
        f[ph] |= r.integers(0, 1 << 63, size=int(ph.sum()), dtype=np.uint64)
    return place


EDGE_CASES = ["one_variable_fills_a_column", "all_self_loops", "all_placeholders", "one_column_of_placeholders",
              "first_and_last_cell_in_one_group", "indices_at_the_ends_and_equal_low_32_bits", "junk_in_bits_48_to_62",
              "placeholders_with_low_bits"]


@pytest.mark.parametrize("name", EDGE_CASES)
def test_sigma_edge_cases(bj, ctx, name):
    place = _edge_case(name)
    got = check_sigma(bj, ctx, place)
    if name in ("all_self_loops", "all_placeholders"):
        assert np.array_equal(got, O.create_permutation_polys(np.full_like(place, PH)))   # sigma = identity
    if name in ("junk_in_bits_48_to_62", "placeholders_with_low_bits"):
        assert np.array_equal(got, O.create_permutation_polys(placement(1, 16)))


@pytest.mark.parametrize("n_cols,log_n", [(128, 24), (1, 31), (2, 30), (256, 23), (155, 24), (3, 30), (1, 33)])
def test_sigma_refuses_2_pow_31_cells_before_allocating(bj, ctx, n_cols, log_n):
    """n_cols * 2^log_n >= 2^31 is refused on the arguments alone: a one-cell buffer stands in for the placement and the
    output, and nothing is launched"""
    import ctypes
    one = bj.to_device(np.zeros(1, np.uint64))
    before = ctx.launch_count()
    st = bj.native.lib.bj_create_permutation_polys(ctx._h, ctypes.c_void_p(one.data_ptr()), n_cols, log_n,
                                                   ctypes.c_void_p(one.data_ptr()))
    assert st == bj.native.BJ_ERR_INVALID_ARG
    assert ctx.launch_count() == before


# ------------------------------------------------------------------------------------------------- witness columns -----
N_VALUES = 1 << 24


def witness_inputs(hint_rows, seed=11):
    """(all_values, hint [V, hint_rows]) at 2^20 rows: values below 2^32 - 1 for a third of them, p added to a seeded share
    of those (non-canonical words of the same field elements), 10 % placeholder cells with junk in their low bits"""
    r = np.random.default_rng(seed)
    values = O.random_field(r, N_VALUES)
    small = r.random(N_VALUES) < 0.3
    values[small] >>= np.uint64(33)
    values[small & (r.random(N_VALUES) < 0.5)] += np.uint64(P)
    values[:4] = [P, P + 1, 2**64 - 1, 2**64 - 2]
    hint = r.integers(0, N_VALUES, size=(V, hint_rows), dtype=np.uint64)
    hint.reshape(-1)[:4] = [0, 1, 2, 3]
    ph = r.random((V, hint_rows)) < 0.1
    ph[0, :4] = False
    hint[ph] = np.uint64(PH) | (hint[ph] & np.uint64(0xFFFF))
    return values, hint


def _non_canonical_cells(values, hint):
    h = hint.reshape(-1)
    live = (h & np.uint64(PH)) == 0
    return int((values[h[live]] >= np.uint64(P)).sum())


def production_columns(bj, log_n):
    """(constants [8, n], lookup dict with tables [4, n], gates) of the production-shaped synthetic circuit, on the host; the
    setup tests bring their own sigma columns"""
    if log_n not in _PRODUCTION:
        from era_boojum_b200 import synthetic
        c = bj.Context(0)
        g = synthetic.generate_production_shaped(c, log_n, seed=70 + log_n)
        lk = dict(g["lookup"])
        lk["tables"] = bj.to_numpy(lk["tables"])
        lk.pop("multiplicities")
        _PRODUCTION[log_n] = (bj.to_numpy(g["constants"]), lk, g["gates"])
        del g
        c.synchronize()
        c.close()
    return _PRODUCTION[log_n]


def _lookup_on_device(bj, lk):
    d = dict(lk)
    d["tables"] = bj.to_device(lk["tables"])
    return d


@pytest.mark.parametrize("hint_rows", [N20, N20 - 1, 1])
def test_witness_columns_2p20(bj, hint_rows):
    """bj_materialize_columns (u64 hint on the device) and bj_setup_attach_variables_hint + bj_witness_upload_vec (u32 hint on
    the setup, all_values uploaded into a slot) both give the oracle's columns: placeholders and rows past hint_rows zero,
    non-canonical values reduced; the u32 multiplicities (n_mult < n, up to 2^32 - 1) are widened and zero-padded.  Then
    bj_materialize_columns refuses the same hint with an index past all_values in its last cell."""
    from era_boojum_b200 import prover
    values, hint = witness_inputs(hint_rows)
    assert hint_rows < 8 or _non_canonical_cells(values, hint) > 1000
    want, bad = O.materialize_columns(values, hint, 20)
    assert bad == 0
    constants, lk, gates = production_columns(bj, 20)
    r = np.random.default_rng(14)
    n_mult = N20 - 12345
    mult = r.integers(0, 2**32, size=n_mult, dtype=np.uint64).astype(np.uint32)
    mult[:2] = [2**32 - 1, 0]
    cfg = prover.ProofConfig(fri_lde_factor=2, merkle_tree_cap_size=32, security_level=100)
    ctx = bj.Context(0)
    try:
        got = bj.to_numpy(ctx.materialize_variables_polynomials_from_dense_hint(bj.to_device(values), bj.to_device(hint), 20))
        assert not _first_difference(got, want), _first_difference(got, want)
        del got
        # the recompute plan keeps the setup small; the gather does not depend on the plan
        mp = bj.proof_memory_plan(20, V, 8, 8, cfg, lookup=lk)
        ctx.allow_recompute_plan(True)
        ctx.set_memory_limit(mp["recompute"] + 2 * bj.witness_slots_bytes(20, V, 1, N_VALUES, lookup=lk))
        sig = bj.to_device(np.zeros((V, N20), np.uint64))   # any sigma columns: the gather does not read them
        nat = ctx.native_setup(sig, bj.to_device(constants), gates, 8, cfg, lookup=_lookup_on_device(bj, lk))
        nat.attach_variables_hint(hint)
        slots = nat.witness_slots(1, N_VALUES)
        slots.upload_vec(0, values, mult)
        got_v, got_m = slots.columns(0)
        assert not _first_difference(got_v, want), _first_difference(got_v, want)
        assert np.array_equal(got_m[:n_mult], mult.astype(np.uint64)) and not got_m[n_mult:].any()
        slots.close()
        nat.close()
        del got_v, got_m, sig
        hint[V - 1, -1] = N_VALUES
        assert O.materialize_columns(values, hint, 20)[1] == 1
        with pytest.raises(bj.BoojumError) as e:
            ctx.materialize_variables_polynomials_from_dense_hint(bj.to_device(values), bj.to_device(hint), 20)
        assert e.value.status == bj.native.BJ_ERR_INVALID_ARG
    finally:
        ctx.close()
        import torch
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------- setup cap -----
def blake2s_cap(cols, cap_size):
    """MerkleTreeWithCap over Blake2s256 (leaf = the LE bytes of one element of every column, node = left | right), the
    recipe of oracle/replay.py::merkle_tree_with_hasher with one hashlib call per leaf on a row-major copy"""
    rows = np.ascontiguousarray(np.asarray(cols, dtype=np.uint64).T)
    width = rows.shape[1] * 8
    mv = memoryview(rows).cast("B")
    cur = b"".join(hashlib.blake2s(mv[i * width:(i + 1) * width], digest_size=32).digest() for i in range(rows.shape[0]))
    while len(cur) > 32 * cap_size:
        cur = b"".join(hashlib.blake2s(cur[64 * i:64 * i + 64], digest_size=32).digest() for i in range(len(cur) // 64))
    return np.frombuffer(cur, dtype="<u8").reshape(-1, 4).copy()


def oracle_cap(cols, log_l, cap_size, hasher):
    """the setup oracle's cap (oracle/prover.py's recipe): the LDE of sigmas | constants | tables over the first L cosets,
    one leaf per point of every column"""
    lde = O.lde(cols, log_l)
    flat = lde.reshape(lde.shape[0], -1)
    if hasher == "poseidon2":
        return O.merkle_tree([flat[c] for c in range(flat.shape[0])], cap_size)[2]
    return blake2s_cap(flat, cap_size)


def test_blake2s_cap_helper_equals_the_oracle_tree():
    r = np.random.default_rng(3)
    cols = O.random_field(r, (5, 64))
    assert np.array_equal(blake2s_cap(cols, 4), R.merkle_tree_with_hasher(list(cols), 4, 1, "blake2s")[2])


# the compact plan needs a quotient degree below the LDE factor, so it runs at L = 8, Q = 4; the other plans run on the
# production geometry L = 2, Q = 8
@pytest.mark.parametrize("log_n,L,Q,hasher,plan", [
    (16, 2, 8, "poseidon2", "resident"),
    (16, 2, 8, "poseidon2", "streamed"),
    (16, 2, 8, "poseidon2", "recompute"),
    (16, 2, 8, "blake2s", "resident"),
    (16, 8, 4, "blake2s", "compact"),
    (20, 2, 8, "blake2s", "resident"),
    (20, 2, 8, "blake2s", "streamed"),
    (20, 2, 8, "blake2s", "recompute"),
])
def test_setup_cap_from_placement_equals_the_oracle(bj, log_n, L, Q, hasher, plan):
    """placement -> bj_create_permutation_polys -> bj_setup_create -> bj_setup_get_cap equals the cap of the oracle's sigma
    columns with the same constants and tables, on every memory plan (each builds the setup tree its own way)"""
    from era_boojum_b200 import prover
    constants, lk, gates = production_columns(bj, log_n)
    place, want_sigma = production_sigma(log_n)
    key = (log_n, L, hasher)
    if key not in _CAPS:
        _CAPS[key] = oracle_cap(np.concatenate([want_sigma, constants, lk["tables"]]), L.bit_length() - 1, 32, hasher)
    cfg = prover.ProofConfig(fri_lde_factor=L, merkle_tree_cap_size=32, security_level=100, hasher=hasher, transcript=hasher)
    ctx = bj.Context(0)
    try:
        mp = bj.proof_memory_plan(log_n, V, 8, Q, cfg, lookup=lk)
        if plan == "recompute":
            ctx.allow_recompute_plan(True)
        ctx.set_memory_limit(mp[plan])
        sig = ctx.create_permutation_polys(bj.to_device(place))
        assert np.array_equal(bj.to_numpy(sig), want_sigma)
        nat = ctx.native_setup(sig, bj.to_device(constants), gates, Q, cfg, lookup=_lookup_on_device(bj, lk))
        assert nat.plan == plan
        got = nat.get_cap()
        assert got.shape == (32, 4) and np.array_equal(got, _CAPS[key]), (log_n, L, hasher, plan)
        nat.close()
    finally:
        ctx.close()
