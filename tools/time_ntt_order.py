"""A/B timing of the NTT tile passes' work order in one process: BJ_NTT_COL_FASTEST = 0 (every pass tile-fastest: one
column's tiles, then the next column's), 1 (front passes column-fastest), 2 (last passes column-fastest, the default) and
3 (both).  One context per setting (the switch is read when a context is created); the settings alternate round by round on
the same 1 GiB batches of bench.py's sweep, forward with coset 7 and without, CUDA-event timed; per-pass kernel times of
the coset-7 transform come from torch.profiler.

    python tools/time_ntt_order.py [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import era_boojum_b200 as bj  # noqa: E402

MODES = (0, 1, 2, 3)


def make_ctx(mode):
    old = os.environ.get("BJ_NTT_COL_FASTEST")
    os.environ["BJ_NTT_COL_FASTEST"] = str(mode)
    try:
        return bj.Context.on_current_stream(0)
    finally:
        if old is None:
            del os.environ["BJ_NTT_COL_FASTEST"]
        else:
            os.environ["BJ_NTT_COL_FASTEST"] = old


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def pass_ms(fn, reps=3):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "ntt_pass" in e.name]
    n = len(kern) // reps
    return [round(sum(kern[r * n + i].device_time_total for r in range(reps)) / reps / 1000.0, 4) for i in range(n)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    ctxs = {m: make_ctx(m) for m in MODES}
    res = {"card": torch.cuda.get_device_name(0), "ms": {}, "pass_ms_coset7": {}}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        res["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception as e:
        res["power_limit_w"] = "unavailable (%s)" % type(e).__name__
    for m in (20, 21, 22, 23, 24):
        d = torch.randint(0, 2**63 - 1, (1 << (27 - m), 1 << m), dtype=torch.int64, device="cuda:0")
        for coset in (7, 1):
            runs = {k: [] for k in MODES}
            for _ in range(args.rounds):
                for k, c in ctxs.items():
                    runs[k].append(timed(lambda: c.fft_natural_to_bitreversed(d, coset)))
            res["ms"]["2^%d_coset%d" % (m, coset)] = {k: round(sorted(v)[len(v) // 2], 4) for k, v in runs.items()}
        res["pass_ms_coset7"]["2^%d" % m] = {k: pass_ms(lambda: c.fft_natural_to_bitreversed(d, 7)) for k, c in ctxs.items()}
        del d
    tot = {k: sum(v[k] for kk, v in res["ms"].items() if kk.endswith("coset7")) for k in MODES}
    res["sweep_coset7_gelem_s"] = {k: round(5 * (1 << 27) / t / 1e6, 2) for k, t in tot.items()}
    for c in ctxs.values():
        c.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
