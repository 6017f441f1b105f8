"""What the timing scripts share: the HBM peak their byte counts are compared with, the device line, the two clocks and
the JSON line of one case.  Nothing here imports torch: the scripts pass it in, so this module imports without a GPU."""
from __future__ import annotations

import json
import subprocess
import time

import numpy as np

PEAK = 3.35e12      # H100 SXM data-sheet HBM3 bandwidth, bytes/s


def device_info(torch):
    """The device name and its power limit (W, None when nvidia-smi cannot be read), read in the same run."""
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return info


def event_times(torch, fn, repeats):
    """Seconds of each of `repeats` calls of fn between two CUDA events on the current stream, after one warm-up
    call."""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return ts


def host_times(torch, fn, repeats):
    """Seconds of each of `repeats` calls of fn on the host clock, after one warm-up call.  The device is synchronised
    before the clock starts and before it is read, so a time holds all the device work the call queued."""
    fn()
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return ts


def line(case, rows, groups, ts, nbytes=None, **extra):
    """Print one case as a JSON line: the median and range of the times `ts` (s) in ms and, given the bytes the case
    must move, those bytes in GB and the fraction of PEAK they would take at the median time."""
    d = {"case": case, "rows": rows, "groups": groups, "ms_median": float(np.median(ts)) * 1e3,
         "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}
    if nbytes is not None:
        d.update({"gbytes": nbytes / 1e9, "hbm_fraction": nbytes / float(np.median(ts)) / PEAK})
    d.update(extra)
    print(json.dumps(d), flush=True)
