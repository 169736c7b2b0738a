"""The cost of one m64nNk16 wgmma (A from registers) for N = 32, 64, 128 at 2 and 3 CTAs per SM, on the skeleton of the
fused solve's field product at config 3's grid (scripts/wgmma_probe.cu: 1,024 CTAs of one warpgroup, 1,020 stages, six
split products over 256 columns per stage).  "resident" is the occupancy the runtime reports: the probe's registers
allow 3 CTAs per SM only at N = 32.  Prints one JSON line: the median CUDA-event time of each configuration, the
SM clocks per wgmma on the busiest SM derived from it, and the card name, power limit, SM clock and throttle reasons
read by nvidia-smi while the probe runs.  Needs the library that `make -C torchcde_b200/csrc` builds beside this file."""
import ctypes
import json
import math
import os
import subprocess
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
N_CTAS, STAGES, PRODUCTS, COLS = 1024, 1020, 6, 256


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return [v.strip() for v in out.split(",")]


def main():
    lib = ctypes.CDLL(os.path.join(HERE, "libwgmma_probe.so"))
    lib.wgmma_probe.argtypes = [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)]
    name, power_limit, sms = smi("name,power.limit,clocks.max.sm")[:3]
    samples, throttles, stop = [], set(), threading.Event()

    def sampler():
        while not stop.is_set():
            clk, thr = smi("clocks.sm,clocks_throttle_reasons.active")[:2]
            samples.append(int(clk))
            throttles.add(thr)
            stop.wait(0.2)

    reps = 5
    rows = []
    th = threading.Thread(target=sampler)
    th.start()
    try:
        for n in (32, 64, 128):
            for per_sm in (2, 3):
                ms = (ctypes.c_float * reps)()
                resident = ctypes.c_int(0)
                rc = lib.wgmma_probe(n, per_sm, N_CTAS, STAGES, reps, ms, ctypes.byref(resident))
                if rc != 0:
                    raise RuntimeError("wgmma_probe(N={}, {} per SM) failed with code {}".format(n, per_sm, rc))
                rows.append((n, per_sm, resident.value, sorted(ms)[reps // 2], min(ms), max(ms)))
    finally:
        stop.set()
        th.join()
    clock = sorted(samples)[len(samples) // 2] if samples else int(sms)
    import torch  # only for the SM count (after the probe, so that its start-up stays out of the clock samples)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    busiest = math.ceil(N_CTAS / n_sm)                     # tiles on the busiest SM
    table = []
    for n, per_sm, resident, med, lo, hi in rows:
        wgmmas = busiest * STAGES * PRODUCTS * (COLS // n)   # per SM
        clk_per = med * 1e-3 * clock * 1e6 / wgmmas
        table.append({"N": n, "ctas_per_sm": per_sm, "resident": resident, "ms": round(med, 3),
                      "ms_range": [round(lo, 3), round(hi, 3)], "clocks_per_wgmma": round(clk_per, 2),
                      "clocks_per_32_columns": round(clk_per * 32 / n, 2)})
    print(json.dumps({"device": name, "power_limit_W": power_limit, "clocks_max_sm_MHz": sms,
                      "clocks_sm_MHz_median": clock, "clocks_sm_MHz_range": [min(samples), max(samples)] if samples else None,
                      "throttle_reasons": sorted(throttles), "sms": n_sm, "probe": table}))


if __name__ == "__main__":
    main()
