"""A/B timing of the forward coset transform's two paths in one process: BJ_NTT_TWIST = 0 (the first pass multiplies every
element by its coset power on load) and 1 (the coset folded into per-round twisted twiddles, the default).  One context per
setting (the switch is read when a context is created); the settings alternate round by round, CUDA-event timed, on:
  - the 1 GiB batches of bench.py's sweep (2^20..2^24), forward on coset 7 and on no coset (which must not move), with the
    per-pass kernel times of the coset-7 transform from torch.profiler;
  - the LDE x2 / x4 / x8 of 16 columns of 2^22 (an inverse, then one forward coset transform per coset);
  - the inverse of 2^22 x 32 columns on coset 7 (untouched by the switch: it must not move).
Card name, power limit and SM clock are read in the same run.

    python tools/time_ntt_twist.py [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import era_boojum_b200 as bj  # noqa: E402

MODES = (0, 1)


def make_ctx(mode):
    old = os.environ.get("BJ_NTT_TWIST")
    os.environ["BJ_NTT_TWIST"] = str(mode)
    try:
        return bj.Context.on_current_stream(0)
    finally:
        if old is None:
            del os.environ["BJ_NTT_TWIST"]
        else:
            os.environ["BJ_NTT_TWIST"] = old


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


def ab(ctxs, rounds, make_fn):
    """median ms per mode, the modes alternating round by round"""
    runs = {k: [] for k in MODES}
    for _ in range(rounds):
        for k, c in ctxs.items():
            runs[k].append(timed(make_fn(c)))
    return {k: {"median": round(sorted(v)[len(v) // 2], 4), "all": [round(x, 4) for x in v]} for k, v in runs.items()}


def card_info():
    info = {"card": torch.cuda.get_device_name(0)}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        info["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        info["sm_clock_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
        info["sm_clock_now_mhz"] = pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception as e:
        info["nvml"] = "unavailable (%s)" % type(e).__name__
    return info


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    ctxs = {m: make_ctx(m) for m in MODES}
    res = {**card_info(), "ms": {}, "pass_ms_coset7": {}}
    for m in (20, 21, 22, 23, 24):
        d = torch.randint(0, 2**63 - 1, (1 << (27 - m), 1 << m), dtype=torch.int64, device="cuda:0")
        for coset in (7, 1):
            res["ms"]["fwd_2^%d_coset%d" % (m, coset)] = ab(ctxs, args.rounds, lambda c: lambda: c.fft_natural_to_bitreversed(d, coset))
        res["pass_ms_coset7"]["2^%d" % m] = {k: pass_ms(lambda: c.fft_natural_to_bitreversed(d, 7)) for k, c in ctxs.items()}
        del d
    d = torch.randint(0, 2**63 - 1, (16, 1 << 22), dtype=torch.int64, device="cuda:0")
    for lde in (2, 4, 8):
        out = torch.empty((16, lde, 1 << 22), dtype=torch.int64, device="cuda:0")
        res["ms"]["lde_2^22x16_x%d" % lde] = ab(ctxs, args.rounds, lambda c: lambda: c.transform_raw_storages_to_lde(d, lde, out=out))
        del out
    d = torch.randint(0, 2**63 - 1, (32, 1 << 22), dtype=torch.int64, device="cuda:0")
    res["ms"]["inv_2^22x32_coset7"] = ab(ctxs, args.rounds, lambda c: lambda: c.ifft_natural_to_natural(d, 7))
    del d
    tot = {k: sum(v[k]["median"] for kk, v in res["ms"].items() if kk.startswith("fwd") and kk.endswith("coset7")) for k in MODES}
    res["sweep_coset7_ms"] = {k: round(t, 4) for k, t in tot.items()}
    res["sweep_coset7_gelem_s"] = {k: round(5 * (1 << 27) / t / 1e6, 2) for k, t in tot.items()}
    res["sm_clock_after_mhz"] = card_info().get("sm_clock_now_mhz")
    for c in ctxs.values():
        c.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
