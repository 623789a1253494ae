"""Witness slot sets without a GPU: bj_witness_slots_bytes against the slot set's pool allocations listed one by one, the
u32 conversion of the variables copy hint (DenseVariablesCopyHint, src/cs/implementations/witness.rs:325-385), and a
restatement of the device gather through the u32 hint against bj_materialize_columns' definition over the u64 hint."""
import numpy as np
import pytest

PLACEHOLDER64 = 1 << 63
PLACEHOLDER32 = 0xFFFFFFFF
P = 0xFFFFFFFF00000001


@pytest.fixture(scope="module")
def bj():
    import era_boojum_b200 as m
    return m


def _pool(n_u64):
    return 8 * max(n_u64, 1)


def _slot_allocations(log_n, V, n_slots, max_values, lookup):
    """the pool allocations bj_witness_slots_create makes (u64 counts), and with max_values > 0 the u32 hint at n rows that
    bj_setup_attach_variables_hint makes"""
    n, lk = 1 << log_n, 1 if lookup else 0
    out = [n_slots * (V + lk) * n]
    if max_values:
        out.append(max_values)
        out.append((V * n + 1) // 2)
        if lookup:
            out.append((n + 1) // 2)
    return out


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("lookup", [None, dict(width=3, num_repetitions=8)])
@pytest.mark.parametrize("max_values", [0, 1, 12345, 1 << 22])
@pytest.mark.parametrize("n_slots", [1, 2, 4])
def test_slot_bytes_replay_the_allocations(bj, world, lookup, max_values, n_slots):
    for log_n, V in ((10, 20), (20, 155), (21, 92)):
        got = bj.witness_slots_bytes(log_n, V, n_slots, max_values, lookup=lookup, world=world)
        want = sum(_pool(a) for a in _slot_allocations(log_n, V, n_slots, max_values, lookup))
        assert got == want, (log_n, V, got, want)


def test_slot_bytes_of_the_production_shape(bj):
    # 2^20 rows, 155 columns + multiplicities: 1.31 GB a slot, and the u32 hint is half the u64 one
    one = bj.witness_slots_bytes(20, 155, 1, 0, lookup=dict(width=3, num_repetitions=8))
    assert one == 156 * 8 << 20
    two_vec = bj.witness_slots_bytes(20, 155, 2, 155 << 20, lookup=dict(width=3, num_repetitions=8))
    assert two_vec == 2 * one + (155 << 23) + (155 << 22) + (1 << 22)


@pytest.mark.parametrize("n_slots,world", [(0, 1), (5, 1), (2, 3), (2, 0)])
def test_slot_bytes_refuses_bad_arguments(bj, n_slots, world):
    with pytest.raises(bj.BoojumError) as e:
        bj.witness_slots_bytes(10, 20, n_slots, 0, world=world)
    assert e.value.status == bj.native.BJ_ERR_INVALID_ARG


def test_hint_u32_conversion(bj):
    h = np.array([[0, 5, PLACEHOLDER64, PLACEHOLDER64 | 7], [(1 << 32) - 2, 3, 1, PLACEHOLDER64]], dtype=np.uint64)
    out, need = bj.variables_hint_to_u32(h)
    assert out.dtype == np.uint32 and out.shape == h.shape
    assert out.tolist() == [[0, 5, PLACEHOLDER32, PLACEHOLDER32], [(1 << 32) - 2, 3, 1, PLACEHOLDER32]]
    assert need == (1 << 32) - 1
    _, need = bj.variables_hint_to_u32(np.full((2, 3), PLACEHOLDER64, np.uint64))
    assert need == 0


@pytest.mark.parametrize("index", [(1 << 32) - 1, 1 << 32, (1 << 48) - 1])
def test_hint_u32_conversion_refuses_an_oversize_index(bj, index):
    h = np.array([[1, 2, index, 3]], dtype=np.uint64)
    with pytest.raises(bj.BoojumError) as e:
        bj.variables_hint_to_u32(h)
    assert e.value.status == bj.native.BJ_ERR_INVALID_ARG


def _materialize_u64(values, hint, n):
    """bj_materialize_columns' definition: out[c][row] = values[hint[c][row]] (reduced) for row < hint_rows; placeholders and
    later rows are zero"""
    out = np.zeros((hint.shape[0], n), np.uint64)
    for c in range(hint.shape[0]):
        for r in range(hint.shape[1]):
            h = int(hint[c, r])
            if not h & PLACEHOLDER64:
                out[c, r] = int(values[h & ((1 << 48) - 1)]) % P
    return out


def _gather_u32(values, hint32, n):
    """the device gather of bj_witness_upload_vec (gather_columns_u32_kernel), one thread per output element"""
    n_cols, hint_rows = hint32.shape
    flat = np.zeros(n_cols * n, np.uint64)
    for i in range(n_cols * n):
        c, row = divmod(i, n)
        if row < hint_rows:
            h = int(hint32[c, row])
            if h != PLACEHOLDER32:
                flat[i] = int(values[h]) % P
    return flat.reshape(n_cols, n)


@pytest.mark.parametrize("seed", range(4))
def test_u32_gather_equals_the_u64_materialisation(bj, seed):
    rng = np.random.default_rng(seed)
    log_n = 6
    n, n_cols = 1 << log_n, 5
    hint_rows = [n, n - 7, 1, 33][seed]
    n_values = 300
    values = rng.integers(0, 1 << 64, n_values, dtype=np.uint64)
    values[:4] = [P, P + 5, (1 << 64) - 1, 0]                         # non-canonical values are reduced by both
    hint = rng.integers(0, n_values, (n_cols, hint_rows)).astype(np.uint64)
    hint[rng.random((n_cols, hint_rows)) < 0.3] = PLACEHOLDER64
    hint[0, 0] = 1                                                     # at least one non-canonical value is read
    hint32, need = bj.variables_hint_to_u32(hint)
    assert need <= n_values
    assert np.array_equal(_gather_u32(values, hint32, n), _materialize_u64(values, hint, n))
