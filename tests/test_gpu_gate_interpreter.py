"""The gate interpreter (csrc/gates.cu) against the C oracle of the recorded programs (orc_gates_quotient / orc_gates_check,
oracle/oracle.c), every output over the whole vector unless stated otherwise, outputs checked canonical.

  * a seeded generator of gate programs that produces every step code (0-47 and the linear combination 48), the peephole's
    aliases, multiply-adds with immediates below and above 2^32, sums of 15 / 16 / 17 small-immediate products with
    coefficients 2^28 - 1 and 2^28, pushes of columns / immediates / shared temporaries, every column kind with per-repetition
    strides, and a gate on specialised columns;
  * inputs mixing 0, 1, p - 1, p, p + 1, 2^32, 2^32 - 1, 2^63, 2^64 - 1 with random u64, and every input 2^64 - 1;
  * eval mode with 1, 2 and 4 points per thread crossed with the peephole settings and ragged sizes, the default dispatch on
    both sides of its thresholds, the 32 / 128 temporary-slot kernels and the 129-slot refusal, a 32-deep selector path, a
    program in its own buffer (over 128 KiB);
  * the SHA-bench and production-shaped gate sets at scale (2^21 / 2^20 points whole, 2^23 points sampled);
  * check mode (bj_check_satisfied) at 2^17, 2^18, 2^19 rows (1, 2, 4 points per thread on 132 SMs) and with 2 or 4 points
    forced at 2^12, with failures planted on points other than the first of a thread;
  * torch.profiler confirms the gate_eval_kernel / gate_check_kernel instantiation each forced case targets."""
import os
import random
import re

import numpy as np
import pytest

from oracle import oracle as O
from tests import test_satisfiability_cpu as CAT
from tests.test_gate_compiler_cpu import _random_program

pytestmark = pytest.mark.gpu

P = O.P
EPS = (1 << 32) - 1
EDGES = np.array([0, 1, P - 1, P, P + 1, 1 << 32, EPS, 1 << 63, 2**64 - 1], dtype=np.uint64)
PEEPHOLES = (0, 1, 2, 4, 8, 15)
V_, W_, C_, T_, K_, CS_ = 0, 1, 2, 3, 4, 5          # BJ_IDX_*
ADD, DOUBLE, SUB, NEGATE, MUL, SQUARE, INVERSE = range(7)  # BJ_REL_*


# ----------------------------------------------------------------------------------------------------- contexts -----
@pytest.fixture(scope="module")
def bj():
    import torch
    assert torch.cuda.is_available()
    import era_boojum_b200 as bj
    yield bj
    for c in _CTX.values():
        c.synchronize()
        c.close()
    _CTX.clear()


_CTX = {}


def context(bj, k=0, peephole=15):
    """a context with the interpreter's points per thread forced to k (0: chosen by size) and the given peephole passes"""
    key = (k, peephole)
    if key not in _CTX:
        os.environ["BJ_GATE_POINTS_PER_THREAD"], os.environ["BJ_GATE_PEEPHOLE"] = str(k), str(peephole)
        try:
            _CTX[key] = bj.Context.on_current_stream(0)
        finally:
            del os.environ["BJ_GATE_POINTS_PER_THREAD"], os.environ["BJ_GATE_PEEPHOLE"]
    return _CTX[key]


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def default_k(n):
    """the interpreter's points per thread when nothing forces it (gates.cu gate_points_per_thread)"""
    s = sm_count()
    return 4 if n >= s * 4 * 512 else 2 if n >= s * 4 * 256 else 1


def gate_kernels(names, check=False):
    """{(K, S)} of the gate kernels among the profiled names"""
    pat = r"gate_%s_kernel<(\d+), (\d+)>" % ("check" if check else "eval")
    return {tuple(int(x) for x in m.groups()) for m in (re.search(pat, s) for s in names) if m}


def kernels_of(fn, attempts=3):
    """names of the CUDA kernels fn() launches, pooled over several traces (a trace can miss kernels); fn must be repeatable"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    names = []
    for _ in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
        names += [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert names, "the profiler recorded no CUDA kernels"
    return names


# ------------------------------------------------------------------------------------------------------- inputs -----
def lazy_u64(rng, shape, edge_fraction=0.3):
    """random u64 (non-canonical ones included) with a fraction replaced by the edge values"""
    a = rng.integers(0, 2**64, size=shape, dtype=np.uint64)
    mask = rng.random(shape) < edge_fraction
    a[mask] = EDGES[rng.integers(0, len(EDGES), size=int(mask.sum()))]
    return a


def selector_columns(rng, n_path, n):
    """selector constants: mostly 0 / 1 (also as p, p + 1), some random"""
    pick = np.array([0, 1, P, P + 1, 0, 1], dtype=np.uint64)
    a = pick[rng.integers(0, len(pick), size=(n_path, n))]
    rnd = rng.random((n_path, n)) < 0.1
    a[rnd] = rng.integers(0, 2**64, size=int(rnd.sum()), dtype=np.uint64)
    return a


# ---------------------------------------------------------------------------------------------- program generator -----
SMALL = [2, 3, 7, 12345, (1 << 28) - 1]
LARGE = [1 << 28, EPS, 1 << 32, (1 << 32) + 1, P - 1, P, P + 1, 1 << 63, 2**64 - 1]


class _Prog:
    """an SSA program in the recorded form, built step by step"""

    def __init__(self, rnd, cols):
        self.rnd, self.cols, self.rel, self.writes = rnd, cols, [], []   # cols: {kind: operands per repetition}
        self.shared = []                                                  # temporaries read more than once

    def emit(self, op, a, b=None):
        self.rel.append((op, len(self.rel), a, b))
        return (T_, len(self.rel) - 1)

    def col(self, kinds=None):
        kinds = [k for k in (kinds or (V_, W_, C_, CS_)) if self.cols.get(k)]
        k = self.rnd.choice(kinds)
        return (k, self.rnd.randrange(self.cols[k]))

    def imm(self, pool=None):
        return (K_, self.rnd.choice(pool or SMALL + LARGE))

    def operand(self, cls):
        return self.rnd.choice(self.shared) if cls == 0 else self.col() if cls == 1 else self.imm()

    def term(self, x, keep=False):
        """x becomes a quotient term; keep: it is also read later (its push is a MOVE of a shared temporary)"""
        self.writes.append(x)
        if keep and x[0] == T_:
            self.shared.append(x)


def generated_program(rnd, cols, lincomb_leaves=(15, 16, 17)):
    """relations + writes that, over the peephole settings, exercise every step code of the interpreter"""
    p = _Prog(rnd, cols)
    for _ in range(4):                                           # shared temporaries (SUB: left alone by every pass)
        p.shared.append(p.emit(SUB, p.col(), p.col()))
    for op in (ADD, SUB, MUL):                                   # codes 0-26: every (class a, class b)
        for ka in range(3):
            for kb in range(3):
                a, b = p.operand(ka), p.operand(kb)
                if kb == 2 and op != SUB:
                    b = p.imm(LARGE + [2, 3, 7])                 # no alias (x + 0, x * 1, x * 0)
                if ka == 2:
                    a = p.imm(LARGE + [2, 3, 7])
                if ka == 1 and kb == 2 and op == ADD:
                    a = p.col([W_, C_, CS_])                     # a column the linear-combination pass leaves to plain steps
                p.term(p.emit(op, a, b), keep=rnd.random() < 0.3)
    for op in (DOUBLE, NEGATE, SQUARE, INVERSE):                 # codes 27-38
        for ka in range(3):
            p.term(p.emit(op, p.operand(ka)), keep=rnd.random() < 0.3)
    for ka in (0, 1):                                            # multiply-adds 42-47 (the product's only use is the sum)
        for kb in range(3):
            pools = [[1 << 28, EPS, (1 << 32) - 2], [1 << 32, (1 << 32) + 1, 1 << 33, P - 1, 2**64 - 1]] if kb == 2 else [None]
            for pool in pools:
                prod = p.emit(MUL, p.operand(ka), p.imm(pool) if kb == 2 else p.operand(kb))
                other = rnd.choice(p.shared)
                p.term(p.emit(ADD, *((prod, other) if rnd.random() < 0.5 else (other, prod))))
    for m in lincomb_leaves:                                     # sums of small-immediate products: 48
        leaves = []
        for i in range(m):
            x = (V_, i % cols[V_]) if i % 3 else rnd.choice(p.shared + [p.emit(NEGATE, p.col())])
            k = (1 << 28) - 1 if i % 4 else rnd.choice([1 << 28, 3, (1 << 28) - 1])
            leaves.append(p.emit(MUL, x, (K_, k)))
        if m == 16:                                              # a balanced tree
            while len(leaves) > 1:
                leaves = [p.emit(ADD, leaves[i], leaves[i + 1]) for i in range(0, len(leaves), 2)]
            s = leaves[0]
        else:                                                    # a chain
            s = leaves[0]
            for x in leaves[1:]:
                s = p.emit(ADD, s, x)
        s = p.emit(ADD, s, (K_, rnd.choice([2**64 - 1, P - 1, 5])))
        p.term(s)
    for m in (16, 17):                                           # at the 96-bit bound: columns times 2^28 - 1 only (with every
        s = p.emit(MUL, (V_, 0), (K_, (1 << 28) - 1))            # input 2^64 - 1, 16 terms fit in 96 bits, 17 would not)
        for i in range(1, m):
            s = p.emit(ADD, s, p.emit(MUL, (V_, i % cols[V_]), (K_, (1 << 28) - 1)))
        p.term(p.emit(ADD, s, (K_, P - 1)))
    x = rnd.choice(p.shared)                                     # the aliases x*1, 1*x, x*0, x+0, 0+x, x-0
    for op, a, b in ((MUL, x, (K_, 1)), (MUL, (K_, 1), x), (MUL, x, (K_, 0)), (ADD, x, (K_, 0)), (ADD, (K_, 0), x), (SUB, x, (K_, 0))):
        y = p.emit(op, a, b)
        p.term(p.emit(MUL, y, rnd.choice(p.shared)))
        p.term(y)
    p.term(p.emit(SUB, p.imm(), rnd.choice(p.shared)))          # I - T
    p.term(p.emit(MUL, p.imm(), p.imm()))                       # I * I
    for kind in (V_, W_, C_, CS_):                               # pushes of bare columns, immediates, shared temporaries
        if cols.get(kind):
            p.term(p.col([kind]))
    p.term(p.imm())
    p.term((K_, 2**64 - 1))
    p.term(rnd.choice(p.shared))
    return p.rel, p.writes


def generated_gates(seed):
    """[general-purpose gate (3 repetitions, strides on every column kind, shared constants), gate on specialised columns (no
    selector, initial offsets, constants shared by its repetitions), a random program (tests/test_gate_compiler_cpu.py)]
    and the column counts (variables, witnesses, constants) they need"""
    rnd = random.Random(seed)
    rel, wr = generated_program(rnd, {V_: 5, W_: 3, C_: 2, CS_: 2})
    gp = dict(name="generated", relations=rel, writes=wr, num_repetitions=3, variables_offset=5, witnesses_offset=3,
              constants_offset=2, constants_placement_offset=3, selector_path=[True, False, True])
    rel, wr = generated_program(rnd, {V_: 5, W_: 3, C_: 2}, lincomb_leaves=(16,))
    spec = dict(name="specialised", relations=rel, writes=wr, num_repetitions=2, variables_offset=5, witnesses_offset=3,
                constants_offset=0, constants_placement_offset=9, selector_path=[], variables_initial_offset=15,
                witnesses_initial_offset=9)
    rel, wr = _random_program(rnd, 120, 5, 2, 2)
    rp = dict(name="random", relations=rel, writes=wr, num_repetitions=3, variables_offset=5, constants_offset=2,
              constants_placement_offset=1, selector_path=[False])
    return [spec, gp, rp], (25, 15, 11)


def step_codes(records):
    """{(code, pushes its value)} of compiled records (the term records of linear combinations skipped)"""
    steps, i = set(), 0
    while i < len(records):
        w0 = int(records[i][0])
        steps.add((w0 & 0x7F, bool(w0 & 0x80)))
        i += 1 + ((int(records[i][1]) + 3) // 4 if (w0 & 0x7F) == 48 else 0)
    return steps


def n_terms(gates):
    return sum(len(g["writes"]) * g["num_repetitions"] for g in gates)


# ------------------------------------------------------------------------------------------------------ running -----
class Case:
    """host columns, alphas and initial q of one gate set; device copies are made per run"""

    def __init__(self, gates, counts, n, seed, n_path=3, all_ones=False):
        rng = np.random.default_rng(seed)
        nv, nw, nc = counts
        self.gates, self.counts, self.n = gates, counts, n
        if all_ones:
            self.var, self.wit, self.con = (np.full((c, n), 2**64 - 1, np.uint64) for c in counts)
            self.q = np.full((2, n), 2**64 - 1, np.uint64)
            self.alphas = [(2**64 - 1, 2**64 - 1)] * n_terms(gates)
        else:
            self.var, self.wit, self.con = lazy_u64(rng, (nv, n)), lazy_u64(rng, (nw, n)), lazy_u64(rng, (nc, n))
            self.con[:n_path] = selector_columns(rng, n_path, n)
            self.q = lazy_u64(rng, (2, n))
            self.alphas = [tuple(int(x) for x in a) for a in lazy_u64(rng, (n_terms(gates), 2))]
        self._want = None

    def want(self):
        if self._want is None:
            self._want = O.gates_quotient(self.gates, self.var, self.wit, self.con, self.alphas, self.q[0], self.q[1])
        return self._want

    def device(self, bj):
        t = [bj.to_device(a) for a in (self.var, self.wit, self.con)]
        return [[x[i] for i in range(x.shape[0])] for x in t]

    def run(self, bj, ctx, cols=None):
        v, w, c = cols or self.device(bj)
        d0, d1 = bj.to_device(self.q[0]), bj.to_device(self.q[1])
        ctx.evaluate_gates_over_general_purpose_columns(self.gates, v, w, c, self.alphas, d0, d1)
        ctx.synchronize()
        return bj.to_numpy(d0), bj.to_numpy(d1)

    def check(self, bj, ctx, cols=None):
        g0, g1 = self.run(bj, ctx, cols)
        w0, w1 = self.want()
        assert (g0 < np.uint64(P)).all() and (g1 < np.uint64(P)).all(), "non-canonical output"
        bad = np.nonzero((g0 != w0) | (g1 != w1))[0]
        assert bad.size == 0, "n=%d: %d points differ, first %s" % (self.n, bad.size, bad[:8].tolist())

    def kernels(self, bj, ctx, cols=None):
        v, w, c = cols or self.device(bj)
        import torch
        d0 = torch.zeros(self.n, dtype=torch.int64, device="cuda:0")
        d1 = torch.zeros(self.n, dtype=torch.int64, device="cuda:0")
        return gate_kernels(kernels_of(lambda: ctx.evaluate_gates_over_general_purpose_columns(self.gates, v, w, c, self.alphas, d0, d1)))


# ------------------------------------------------------------------------------------------- the generated set -----
def test_generated_programs_cover_every_step_code(bj):
    """host-side: over the peephole settings the generated gate set compiles to every step code 0-48; the default setting
    keeps the multiply-adds, linear combinations and pushing steps"""
    gates, (nv, nw, nc) = generated_gates(0)
    seen = set()
    for pp in PEEPHOLES:
        steps = step_codes(bj.compile_gate_programs(gates, nv, nw, nc, pp)[0])
        seen |= {code for code, _ in steps}
        if pp == 15:
            default = steps
    assert seen == set(range(49)), sorted(set(range(49)) - seen)
    codes = {code for code, _ in default}
    assert set(range(42, 49)) <= codes and set(range(39, 42)) <= codes, sorted(codes)
    assert len({code for code, push in default if push}) >= 20     # steps that push the value they compute


@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("peephole", PEEPHOLES)
def test_eval_sweep(bj, k, peephole):
    """points per thread forced to k, each peephole setting, ragged sizes (1, 127, 129, 511, 513, 128 K m +- 1): every point
    equals the oracle; the profiler sees gate_eval_kernel<k, S>"""
    gates, counts = generated_gates(1)
    ctx = context(bj, k, peephole)
    sizes = [1, 127, 129, 511, 513, 128 * k * 5 - 1, 128 * k * 5 + 1]
    for i, n in enumerate(sizes):
        case = Case(gates, counts, n, seed=10 * i + k)
        case.check(bj, ctx)
    live = bj.compile_gate_programs(gates, *counts, peephole)[2]
    assert case.kernels(bj, ctx) == {(k, 32 if live <= 32 else 128)}


def test_every_input_all_ones(bj):
    """columns, initial q and alphas all 2^64 - 1: the 96-bit linear combinations (16 terms with coefficient 2^28 - 1) and
    the 32-bit immediate paths at their largest operands"""
    gates, counts = generated_gates(2)
    for k in (1, 2, 4):
        for pp in (4, 15):
            Case(gates, counts, 1000, seed=0, all_ones=True).check(bj, context(bj, k, pp))


def test_default_dispatch_thresholds(bj):
    """with nothing forced: 1 point per thread below sm_count * 4 * 256 points, 2 from there, 4 from sm_count * 4 * 512"""
    gates, counts = generated_gates(3)
    ctx = context(bj)
    s = sm_count()
    for n in (s * 4 * 256 - 1, s * 4 * 256, s * 4 * 512 - 1, s * 4 * 512):
        case = Case(gates, counts, n, seed=n)
        cols = case.device(bj)
        case.check(bj, ctx, cols)
        assert {k for k, _ in case.kernels(bj, ctx, cols)} == {default_k(n)}, n


# ---------------------------------------------------------------------------------------------- kernel boundaries -----
def live_program(n_live):
    """n_live products of two variable columns, all live when the first of them is read: a chain of products over them (no
    pass merges products into sums)"""
    rel = [(MUL, i, (V_, i % 7), (V_, (i * 3 + 1) % 7)) for i in range(n_live)]
    s = (T_, 0)
    for i in range(1, n_live):
        rel.append((MUL, len(rel), s, (T_, i)))
        s = (T_, len(rel) - 1)
    return dict(relations=rel, writes=[s, (T_, n_live // 2) if n_live > 1 else s], num_repetitions=2, variables_offset=3,
                constants_offset=0, constants_placement_offset=1, selector_path=[True])


@pytest.mark.parametrize("n_live,slots", [(32, 32), (33, 128), (128, 128)])
def test_live_temporaries(bj, n_live, slots):
    gate = live_program(n_live)
    # temporary n_live // 2 is read twice (the chain, the write): with it the chain's first product still sees all n_live live
    for pp in (0, 15):
        assert bj.compile_gate_programs([gate], 10, 0, 1, pp)[2] == n_live
    for k in (1, 2, 4):
        case = Case([gate], (10, 0, 1), 700, seed=n_live + k, n_path=1)
        ctx = context(bj, k)
        case.check(bj, ctx)
        assert case.kernels(bj, ctx) == {(k, slots)}


def test_129_live_temporaries_are_refused(bj):
    import torch
    gate = live_program(129)
    ctx = context(bj)
    v = [bj.to_device(np.arange(64, dtype=np.uint64)) for _ in range(10)]
    d0 = torch.zeros(64, dtype=torch.int64, device="cuda:0")
    d1 = torch.zeros(64, dtype=torch.int64, device="cuda:0")
    with pytest.raises(bj.BoojumError) as e:
        ctx.evaluate_gates_over_general_purpose_columns([gate], v, [], [bj.to_device(np.ones(64, np.uint64))], [(1, 0)] * 4, d0, d1)
    assert e.value.status == bj.native.BJ_ERR_UNSUPPORTED


def test_selector_path_32_deep(bj):
    """a path of 32 (bit 31 set) over 32 selector columns; rows matching the path (selector 1), rows off it (0), random"""
    rnd = random.Random(5)
    path = [rnd.random() < 0.5 for _ in range(31)] + [True]
    rel, wr = generated_program(rnd, {V_: 5, W_: 3, C_: 2, CS_: 2}, lincomb_leaves=(16,))
    gate = dict(relations=rel, writes=wr, num_repetitions=2, variables_offset=5, witnesses_offset=3, constants_offset=2,
                constants_placement_offset=32, selector_path=path)
    for k in (1, 2, 4):
        case = Case([gate], (10, 6, 36), 1500, seed=k, n_path=32)
        on = np.array([[1 if b else 0] for b in path], np.uint64)
        case.con[:32, ::3] = on                                  # selected rows
        case.con[:32, 1::3] = on
        case.con[31, 1::3] = 0                                   # off by the last bit alone
        case.check(bj, context(bj, k))


def test_program_in_its_own_buffer(bj):
    """a program of more than 4096 records (128 KiB) is uploaded to its own buffer: 1, 2 and 4 points per thread"""
    rnd = random.Random(6)
    rel = [(SUB, 0, (V_, 0), (W_, 0))]
    for i in range(1, 5000):
        op = rnd.choice([ADD, SUB, MUL, MUL, SQUARE, NEGATE])
        b = rnd.choice([(V_, i % 4), (W_, i % 2), (C_, 0), (K_, rnd.choice(SMALL + LARGE))])
        rel.append((op, i, (T_, i - 1), b if op in (ADD, SUB, MUL) else None))
    gate = dict(relations=rel, writes=[(T_, 4999), (T_, 2500)], num_repetitions=2, variables_offset=4, witnesses_offset=2,
                constants_offset=1, constants_placement_offset=0, selector_path=[])
    assert len(bj.compile_gate_programs([gate], 8, 4, 2, 15)[0]) * 32 > 128 << 10
    for k in (1, 2, 4):
        case = Case([gate], (8, 4, 2), 2000, seed=k, n_path=0)
        ctx = context(bj, k)
        case.check(bj, ctx)
        assert {kk for kk, _ in case.kernels(bj, ctx)} == {k}


# ------------------------------------------------------------------------------------------------ production scale -----
def sha_gate_set():
    from era_boojum_b200 import synthetic
    return synthetic.sha_shaped_gates(60), (60, 0, 6), 2


def production_gate_set():
    from tests.test_oracle_prover_cpu import production_gates
    gates = production_gates()[0]
    assert n_terms(gates) == 415
    return gates, (155, 0, 8), 6


def device_columns(n_cols, n, seed):
    """[n_cols, n] random u64 with edge values, generated on the device"""
    import torch
    g = torch.Generator(device="cuda:0")
    g.manual_seed(seed)
    edges = torch.tensor(EDGES.view(np.int64), device="cuda:0")
    out = torch.empty((n_cols, n), dtype=torch.int64, device="cuda:0")
    for c in range(n_cols):
        hi = torch.randint(0, 1 << 32, (n,), dtype=torch.int64, device="cuda:0", generator=g)
        lo = torch.randint(0, 1 << 32, (n,), dtype=torch.int64, device="cuda:0", generator=g)
        col = (hi << 32) | lo
        pick = torch.randint(0, 4 * len(EDGES), (n,), dtype=torch.int64, device="cuda:0", generator=g)
        out[c] = torch.where(pick < len(EDGES), edges[pick.clamp(max=len(EDGES) - 1)], col)
    return out


@pytest.mark.parametrize("which,log_n", [("sha", 21), ("production", 20)])
def test_gate_sets_at_scale(bj, which, log_n):
    """the SHA-bench gate set and the production-shaped one (415 terms, the Poseidon2 flattened gate) over whole vectors,
    default dispatch"""
    import torch
    gates, (nv, nw, nc), n_path = sha_gate_set() if which == "sha" else production_gate_set()
    n = 1 << log_n
    cols = device_columns(nv + nc + 2, n, seed=log_n)
    rng = np.random.default_rng(log_n)
    alphas = [tuple(int(x) for x in a) for a in lazy_u64(rng, (n_terms(gates), 2))]
    sel = torch.tensor(selector_columns(rng, n_path, n).view(np.int64), device="cuda:0")
    cols[nv:nv + n_path] = sel
    q0, q1 = cols[nv + nc].clone(), cols[nv + nc + 1].clone()
    ctx = context(bj)
    ctx.evaluate_gates_over_general_purpose_columns(gates, [cols[i] for i in range(nv)], [], [cols[nv + i] for i in range(nc)],
                                                    alphas, q0, q1)
    ctx.synchronize()
    host = bj.to_numpy(cols)
    got0, got1 = bj.to_numpy(q0), bj.to_numpy(q1)
    del cols, q0, q1, sel
    torch.cuda.empty_cache()
    w0, w1 = O.gates_quotient(gates, host[:nv], [], host[nv:nv + nc], alphas, host[nv + nc], host[nv + nc + 1])
    assert (got0 < np.uint64(P)).all() and (got1 < np.uint64(P)).all()
    bad = np.nonzero((got0 != w0) | (got1 != w1))[0]
    assert bad.size == 0, "%d points differ, first %s" % (bad.size, bad[:8].tolist())


def test_production_gate_set_at_2_23_points_sampled(bj):
    """2^20 rows x Q = 8 = 2^23 points (4 per thread by default): every point of a set of blocks (first, last and some
    between), then random points, against the oracle on the gathered columns"""
    import torch
    gates, (nv, nw, nc), n_path = production_gate_set()
    n = 1 << 23
    k = default_k(n)
    cols = device_columns(nv + nc + 2, n, seed=23)
    rng = np.random.default_rng(23)
    cols[nv:nv + n_path] = torch.tensor(selector_columns(rng, n_path, n).view(np.int64), device="cuda:0")
    alphas = [tuple(int(x) for x in a) for a in lazy_u64(rng, (n_terms(gates), 2))]
    q0, q1 = cols[nv + nc].clone(), cols[nv + nc + 1].clone()
    ctx = context(bj)
    ctx.evaluate_gates_over_general_purpose_columns(gates, [cols[i] for i in range(nv)], [], [cols[nv + i] for i in range(nc)],
                                                    alphas, q0, q1)
    ctx.synchronize()
    block = 128 * k
    n_blocks = n // block
    blocks = sorted({0, 1, n_blocks // 2, n_blocks - 2, n_blocks - 1} | set(rng.integers(0, n_blocks, 3).tolist()))
    idx = np.unique(np.concatenate([np.arange(b * block, (b + 1) * block) for b in blocks] + [rng.integers(0, n, 3000)]))
    ti = torch.tensor(idx, device="cuda:0")
    host = bj.to_numpy(cols[:, ti].contiguous())
    got0, got1 = bj.to_numpy(q0[ti]), bj.to_numpy(q1[ti])
    names = kernels_of(lambda: ctx.evaluate_gates_over_general_purpose_columns(
        gates, [cols[i] for i in range(nv)], [], [cols[nv + i] for i in range(nc)], alphas, q0, q1), attempts=1)
    del cols, q0, q1
    torch.cuda.empty_cache()
    w0, w1 = O.gates_quotient(gates, host[:nv], [], host[nv:nv + nc], alphas, host[nv + nc], host[nv + nc + 1])
    bad = np.nonzero((got0 != w0) | (got1 != w1))[0]
    assert bad.size == 0, "%d sampled points differ, first %s" % (bad.size, idx[bad[:8]].tolist())
    assert {kk for kk, _ in gate_kernels(names)} == {k}


# ---------------------------------------------------------------------------------------------- check mode at scale -----
def selected(gates, con, row):
    """indices of the gates (with terms) whose selector is nonzero on the row"""
    c = [int(x) % P for x in con[:, row]]
    out = []
    for gi, g in enumerate(gates):
        s = 1
        for i, bit in enumerate(g["selector_path"]):
            s = s * (c[i] if bit else 1 - c[i]) % P
        if s and g["writes"]:
            out.append(gi)
    return out


class CheckCircuit:
    """a satisfied circuit generated on the device, its host columns, and mutations that break one gate on one row"""

    def __init__(self, bj, ctx, kind, log_n):
        from era_boojum_b200 import synthetic
        if kind == "sha":
            v, s, c, gates, _, lk = synthetic.generate(ctx, log_n, 60, seed=log_n, lookup=True)
        else:
            d = synthetic.generate_production_shaped(ctx, log_n, seed=log_n)
            v, s, c, gates, lk = d["variables"], d["sigmas"], d["constants"], d["gates"], d["lookup"]
        self.bj, self.kind, self.v, self.s, self.c, self.gates, self.lk = bj, kind, v, s, c, gates, lk
        self.var, self.con = bj.to_numpy(v), bj.to_numpy(c)
        self.n = self.var.shape[1]
        # gates a constant change breaks: general-purpose gates that read a constant column
        self.breakable = [gi for gi, g in enumerate(gates) if g["selector_path"]
                          and any(r[2][0] in (C_, CS_) or (r[3] is not None and r[3][0] in (C_, CS_)) for r in g["relations"])]

    def plant(self, row, gi):
        """break gate gi on the row: + 1 on its first constant column (the boolean gate of the production shape: its column = 2)"""
        g = self.gates[gi]
        if not g["selector_path"]:
            col = g["variables_initial_offset"]
            return ("v", col, row, 2)
        col = g["constants_placement_offset"]
        return ("c", col, row, (int(self.con[col, row]) + 1) % P)

    def report(self, ctx, plants):
        """(device report, oracle report) with the plants applied to copies"""
        v, c = self.v, self.c
        var, con = self.var, self.con
        rows = sorted({r for _, _, r, _ in plants})
        sub_v, sub_c = var[:, rows].copy(), con[:, rows].copy()
        if plants:
            v, c = v.clone(), c.clone()
        for which, col, row, val in plants:
            (v if which == "v" else c)[col, row] = val - 2**64 if val >= 2**63 else val
            (sub_v if which == "v" else sub_c)[col, rows.index(row)] = val
        got = ctx.check_if_satisfied(v, self.s, c, self.gates, lookup=self.lk)
        want = O.gates_report(self.gates, sub_v, sub_c)
        if want["gate_failures"]:
            want["gate_row"] = rows[want["gate_row"]]
        per_row = O.gates_check(self.gates, sub_v, sub_c)
        return got, CAT.expect(**want), {r: int(per_row["first_value"][i]) for i, r in enumerate(rows)}

    def thread_rows(self, k, block, tid):
        return [block * 128 * k + j * 128 + tid for j in range(k)]

    def find_thread(self, k, want_fn, start_block=1):
        """the first thread (block, lane) whose rows satisfy want_fn(list of selected gate sets)"""
        for block in range(start_block, self.n // (128 * k)):
            for tid in range(0, 128, 7):
                rows = self.thread_rows(k, block, tid)
                sel = [selected(self.gates, self.con, r) for r in rows]
                got = want_fn(sel)
                if got is not None:
                    return rows, got
        raise AssertionError("no thread with the wanted row kinds")


def term_base(gates, gi):
    return sum(len(g["writes"]) * g["num_repetitions"] for g in gates[:gi])


def _check_scenarios(bj, ctx, circ, k):
    gates = circ.gates
    breakable = circ.breakable
    got, want, _ = circ.report(ctx, [])
    assert got == want == CAT.expect(), "the generated circuit is not satisfied"
    scenarios = {}
    # 1. one failure on the thread's last point (k >= 1 when K > 1); point 0 passes
    rows, gi = circ.find_thread(k, lambda s: next((g for g in s[-1] if g in breakable), None))
    scenarios["last_point"] = ([circ.plant(rows[-1], gi)], [rows[-1]])
    # 2. a failure on a point k >= 1 whose gate is unselected on point 0 of the thread (the program must still run)
    if k > 1:
        rows, (j, gi) = circ.find_thread(k, lambda s: next(((j, g) for j in range(1, k) for g in s[j] if g in breakable and g not in s[0]), None))
        scenarios["unselected_on_point_0"] = ([circ.plant(rows[j], gi)], [rows[j]])
        # 3. failures on two points of one thread, the later point holding the smaller term index
        rows, (j, g0, g1) = circ.find_thread(k, lambda s: next(((j, a, b) for j in range(1, k) for a in s[0] for b in s[j]
                                                                 if a in breakable and b in breakable
                                                                 and term_base(gates, b) < term_base(gates, a)), None))
        scenarios["later_point_smaller_term"] = ([circ.plant(rows[0], g0), circ.plant(rows[j], g1)], [rows[0], rows[j]])
        # ... and the same with point 0 passing: the later point's value and selector are its own
        scenarios["later_point_alone"] = ([circ.plant(rows[j], g1)], [rows[j]])
    # 4. a thread whose point j does not select a gate that another of its points selects (and passes): the program runs for
    #    point j too and its terms there are nonzero, yet they count nothing (the satisfied circuit reports nothing, above)
    if k > 1:
        rows, (j, gi) = circ.find_thread(k, lambda s: next(((j, g) for j in range(len(s)) for g in breakable
                                                            if g not in s[j] and any(g in t for t in s)), None))
        alone = dict(gates[gi], selector_path=[])
        assert O.gates_check([alone], circ.var[:, rows[j]:rows[j] + 1], circ.con[:, rows[j]:rows[j] + 1])["failures"]
    # 5. the last row
    r = circ.n - 1
    gi = next(g for g in selected(gates, circ.con, r) if g in breakable or not gates[g]["selector_path"])
    scenarios["last_row"] = ([circ.plant(r, gi)], [r])
    for name, (plants, failing) in scenarios.items():
        got, want, first_values = circ.report(ctx, plants)
        assert [r for r, v in sorted(first_values.items()) if v] == failing, (name, first_values)
        assert got == want, (name, got, want)
    names = kernels_of(lambda: ctx.check_if_satisfied(circ.v, circ.s, circ.c, gates, lookup=circ.lk), attempts=2)
    assert {kk for kk, _ in gate_kernels(names, check=True)} == {k}


@pytest.mark.parametrize("kind", ["sha", "production"])
@pytest.mark.parametrize("log_n", [17, 18, 19])
def test_check_mode_at_scale(bj, kind, log_n):
    import torch
    ctx = context(bj)
    circ = CheckCircuit(bj, ctx, kind, log_n)
    full = O.gates_report(circ.gates, circ.var, circ.con)
    assert full["gate_failures"] == 0
    _check_scenarios(bj, ctx, circ, default_k(circ.n))
    del circ
    torch.cuda.empty_cache()


@pytest.mark.parametrize("kind", ["sha", "production"])
@pytest.mark.parametrize("k", [2, 4])
def test_check_mode_forced_points_per_thread(bj, kind, k):
    ctx = context(bj, k)
    circ = CheckCircuit(bj, ctx, kind, 12)
    assert O.gates_report(circ.gates, circ.var, circ.con)["gate_failures"] == 0
    _check_scenarios(bj, ctx, circ, k)
