"""JPEG decoding (sfmb200_decode_jpeg_batch) against cv2.imdecode on the same machine.

    python tools/bench_jpeg.py [--reps 20] [--out results/bench_jpeg.json]

Workloads: the committed crazyhorse JPEG (1024x768 4:2:2, 404 KB, the files runSfM reads) x7 -- one run's images -- and x50 in one call,
and 50 synthetic 4000x3000 q95 4:2:0 files (seeded).  Per workload: host clock around the synchronised call (warmed up; median and
max over repeats), the upload / download bytes and the Huffman counters of the call, cv2.imdecode on one host thread and on all host
threads.  Kernel times come from torch.profiler in a separate pass, split into unstuff, Huffman synchronisation (with the block
prefix sum), Huffman write, DC prediction, IDCT and colour.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import subprocess
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


PHASES = (("unstuff", ("jd_unstuff",)), ("huffman_sync", ("jd_sync", "jd_nblk", "AddU32")), ("huffman_write", ("jd_write",)),
          ("dc_prediction", ("jd_dc_", "Add3x16")), ("idct", ("jd_idct",)), ("colour", ("jd_color",)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    import jpeg_util as J
    from sfm_toy_library_b200 import capi
    ctx = capi.Context(0)
    ch = J.crazyhorse()
    t0 = time.perf_counter()
    big = [J.encode(4000, 3000, q=95, sampling="420", seed=1000 + k) for k in range(50)]
    gen_s = time.perf_counter() - t0
    loads = {"crazyhorse_x7": [ch] * 7, "crazyhorse_x50": [ch] * 50, "synthetic_4000x3000_q95_420_x50": big}
    res = {"metric": "jpeg_decode_ms_per_call", "generation_s": gen_s}
    for name, files in loads.items():
        ref = [cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) for b in files[:3]]
        out = ctx.decode_jpeg(files)
        assert all(np.array_equal(x, y) for x, y in zip(out, ref)), name
        st = ctx.jpeg_last_stats()
        ms = []
        for _ in range(a.reps):
            t0 = time.perf_counter(); ctx.decode_jpeg(files); ms.append(1e3 * (time.perf_counter() - t0))
        bufs = [np.frombuffer(b, np.uint8) for b in files]
        t0 = time.perf_counter()
        for b in bufs:
            cv2.imdecode(b, cv2.IMREAD_COLOR)
        cv1 = 1e3 * (time.perf_counter() - t0)
        with ThreadPoolExecutor(os.cpu_count()) as ex:
            t0 = time.perf_counter(); list(ex.map(lambda b: cv2.imdecode(b, cv2.IMREAD_COLOR), bufs)); cvn = 1e3 * (time.perf_counter() - t0)
        res[name] = {"files": len(files), "input_bytes": int(sum(len(b) for b in files)), "gpu_call_median_ms": float(np.median(ms)),
                     "gpu_call_max_ms": float(np.max(ms)), "cv2_imdecode_1_thread_ms": cv1, "cv2_imdecode_%d_threads_ms" % os.cpu_count(): cvn,
                     "speedup_vs_cv2_1_thread": cv1 / float(np.median(ms)), "call_stats": st,
                     "sync_extra_codewords_per_subsequence": st["codewords_sync"] / max(1, st["subsequences"])}
    for name, files in loads.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ctx.decode_jpeg(files)
        k = {p: 0.0 for p, _ in PHASES}; other = 0.0
        for e in prof.events():
            t = 1e-3 * e.device_time_total
            for p, keys in PHASES:
                if any(x in e.name for x in keys):
                    k[p] += t; break
            else:
                if "jd_" in e.name or "scan_" in e.name:
                    other += t
        k["total_kernels"] = sum(k.values()) + other
        res[name]["kernel_ms_torch_profiler"] = k
    res["card"], res["power_limit"] = card()
    res["host_threads"] = os.cpu_count()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
