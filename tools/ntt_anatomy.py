"""Anatomy of the forward coset-7 NTT sweep (bench.py's headline workload) on one GPU, in one run:

  - card name, power limit and the SM clock right after the sweep (NVML, read only);
  - cycles per warp-butterfly of tools/ubench/alu_mix.cu (the integer pipes with no memory traffic), compiled into a
    temporary directory;
  - a 1 GiB device-to-device copy: the memory-only time of one pass (1 GiB read + 1 GiB written);
  - per-pass kernel times of each sweep size (1 GiB of columns, coset 7) from torch.profiler;
  - tools/time_ntt.py's forward time with coset 7 and without a coset (the difference is the coset-power table's cost).

Each pass is set against two models: t_alu (the pass's butterflies at the measured butterfly rate, all SMs busy) and
t_mem (the copy time).  A pass whose time sits near max(t_alu, t_mem) overlaps memory and compute already; one near
t_alu + t_mem runs them one after the other.  Env toggles of the library (BJ_NTT_*) apply.

    python tools/ntt_anatomy.py [--out FILE]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import era_boojum_b200 as bj  # noqa: E402

SIZES = (20, 21, 22, 23, 24)
BATCH_LOG = 27  # 1 GiB of u64 per size, as in bench.py
COSET = 7


def card():
    out = {"name": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        out["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
        out["_nvml"] = (pynvml, h)
    except Exception as e:  # the numbers stand without it, but say so
        out["nvml"] = "unavailable (%s)" % type(e).__name__
    return out


def sm_clock(c):
    if "_nvml" not in c:
        return None
    nv, h = c["_nvml"]
    return nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)


def alu_bfly():
    """cycles per warp-butterfly of alu_mix's `bfly x8` line, per resident CTAs of 256 threads per SM"""
    src = os.path.join(ROOT, "tools", "ubench", "alu_mix.cu")
    inc = os.path.join(ROOT, "era_boojum_b200", "csrc")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "alu_mix")
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", exe, src, "-I", inc])
        text = subprocess.check_output([exe], text=True)
    res = {}
    for line in text.splitlines():
        mt = re.match(r"ctas/SM (\d+)\s+bfly x8: ([\d.]+) Gbfly/s \(([\d.]+) SMSP-cycles per warp-butterfly\)", line)
        if mt:
            res[int(mt.group(1))] = {"gbfly_s": float(mt.group(2)), "smsp_cycles_per_warp_bfly": float(mt.group(3))}
    return res


def events_ms(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def copy_ms():
    x = torch.empty(1 << BATCH_LOG, dtype=torch.int64, device="cuda:0")
    y = torch.empty_like(x)
    x.fill_(1)
    t = events_ms(lambda: y.copy_(x), 10)
    del x, y
    return t


def per_pass(ctx, m, reps=3):
    """device ms of each pass kernel of one forward coset-7 transform of 2^(27-m) columns of 2^m, in launch order"""
    from torch.profiler import ProfilerActivity, profile
    cols = 1 << (BATCH_LOG - m)
    d = torch.randint(0, 2**63 - 1, (cols, 1 << m), dtype=torch.int64, device="cuda:0")
    for _ in range(2):
        ctx.fft_natural_to_bitreversed(d, COSET)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ctx.fft_natural_to_bitreversed(d, COSET)
        torch.cuda.synchronize()
    del d
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "ntt_pass" in e.name]
    n_pass = len(kern) // reps
    out = []
    for i in range(n_pass):
        ts = [kern[r * n_pass + i] for r in range(reps)]
        out.append({"kernel": ts[0].name, "ms": round(sum(e.device_time_total for e in ts) / reps / 1000.0, 4)})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", help="also write the JSON here")
    args = ap.parse_args()
    c = card()
    bfly = alu_bfly()
    ctx = bj.Context.on_current_stream(0)
    t_copy = copy_ms()
    sizes = {}
    for m in SIZES:
        sizes["2^%d" % m] = per_pass(ctx, m)
    clk1 = sm_clock(c)
    ctx.close()
    tn = subprocess.check_output([sys.executable, os.path.join(ROOT, "tools", "time_ntt.py")], text=True)
    time_ntt = json.loads(tn.strip().splitlines()[-1])

    # t_alu of a pass of t rounds: 2^26 * t butterflies = 2^21 * t warp-butterflies over 4 SMSPs per SM, at the butterfly rate
    # of 4 resident CTAs of 256 threads per SM (the measured occupancy nearest the 3 of the 2^13-value tiles)
    mhz = clk1 or c.get("sm_max_mhz")
    occ = 4 if 4 in bfly else (max(bfly) if bfly else None)
    cyc = bfly[occ]["smsp_cycles_per_warp_bfly"] if occ else None
    smsps = 4 * c["sms"]
    for key, passes in sizes.items():
        for p in passes:
            mt = re.search(r"<(\d+), (\d+), (\d+)>", p["kernel"])
            t = int(mt.group(1)) if mt else None
            p["t"] = t
            if t and cyc and mhz:
                t_alu = ((1 << 21) * t * cyc / smsps) / (mhz * 1e6) * 1e3
                p["t_alu_ms"] = round(t_alu, 4)
                p["t_mem_ms"] = round(t_copy, 4)
                p["vs_max"] = round(p["ms"] / max(t_alu, t_copy), 3)
                p["vs_sum"] = round(p["ms"] / (t_alu + t_copy), 3)
    c.pop("_nvml", None)
    res = {"card": c, "sm_mhz_after_sweep": clk1, "alu_mix_bfly": bfly, "alu_mix_occupancy_used": occ,
           "copy_1gib_d2d_ms": round(t_copy, 4), "copy_gbs": round(2 * (1 << 30) / t_copy / 1e6, 1), "passes": sizes,
           "time_ntt_gelem_s": time_ntt,
           "env": {k: v for k, v in os.environ.items() if k.startswith("BJ_NTT")}}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
