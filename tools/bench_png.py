"""PNG decoding (sfmb200_decode_images) against cv2.imdecode on the same machine.

    python tools/bench_png.py [--reps 10] [--out results/bench_png.json]

Workloads: the crazyhorse image written by cv2.imencode(".png") at its default level, x7 -- one run's images -- and x50 in one call;
50 seeded synthetic 4000x3000 PNGs; and the crazyhorse PNG written with the Z_FIXED strategy x7, whose fixed-Huffman blocks the chain
decodes serially.  Per workload: host clock around the synchronised call (warmed up; median and max over repeats), cv2.imdecode on one
host thread and on all host threads, png_last_stats, the host parse time (sfmb200_image_info over every file), and the fused
decode_images_orb call (images not downloaded) against cv2.imdecode then orb_detect_and_compute.  Kernel times per phase (scan, probe, chain,
write, rounds, pack + Adler-32, unfilter, colour, resize) come from torch.profiler in a separate pass.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

PHASES = (("scan", ("pg_scan",)), ("probe", ("pg_probe",)), ("chain", ("pg_chain", "pg_block_prefix")), ("write", ("pg_write",)), ("rounds", ("pg_round",)), ("pack_adler", ("pg_pack",)),
          ("unfilter", ("pg_unfilter",)), ("colour", ("pg_color",)), ("resize", ("rz_linear", "rz_area")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--big", type=int, default=50, help="synthetic 4000x3000 files")
    a = ap.parse_args()
    import cv2
    import torch
    import png_util as P
    from bench_jpeg import card
    from sfm_toy_library_b200 import capi
    ctx = capi.Context(0)
    ch = P.crazyhorse()
    chp = P.imencode(ch)
    fixed = P.imencode(ch, [cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_STRATEGY_FIXED])
    t0 = time.perf_counter()
    rs = np.random.RandomState(7)
    big = []
    for k in range(a.big):
        small = rs.randint(0, 256, (300, 400, 3)).astype(np.uint8)
        img = cv2.resize(small, (4000, 3000), interpolation=cv2.INTER_CUBIC)
        img = cv2.add(img, rs.randint(0, 8, img.shape).astype(np.uint8))
        big.append(P.imencode(img))
    gen_s = time.perf_counter() - t0
    loads = {"crazyhorse_png_x7": [chp] * 7, "crazyhorse_png_x50": [chp] * 50, "synthetic_4000x3000_png_x%d" % a.big: big,
             "crazyhorse_png_zfixed_x7": [fixed] * 7}
    res = {"metric": "png_decode_ms_per_call", "generation_s": gen_s}
    for name, files in loads.items():
        ref = [cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) for b in files[:2]]
        out = ctx.decode_images(files)
        assert all(np.array_equal(x, y) for x, y in zip(out, ref)), name
        st = ctx.png_last_stats()
        ms = []
        for _ in range(a.reps):
            t0 = time.perf_counter(); ctx.decode_images(files); ms.append(1e3 * (time.perf_counter() - t0))
        t0 = time.perf_counter()
        for f in files:
            capi.image_info(f)
        parse = 1e3 * (time.perf_counter() - t0)
        bufs = [np.frombuffer(b, np.uint8) for b in files]
        threads = cv2.getNumThreads()
        cv2.setNumThreads(1)
        t0 = time.perf_counter()
        for b in bufs:
            cv2.imdecode(b, cv2.IMREAD_COLOR)
        cv1 = 1e3 * (time.perf_counter() - t0)
        cv2.setNumThreads(threads)
        with ThreadPoolExecutor(os.cpu_count()) as ex:
            t0 = time.perf_counter(); list(ex.map(lambda b: cv2.imdecode(b, cv2.IMREAD_COLOR), bufs)); cvn = 1e3 * (time.perf_counter() - t0)
        r = {"files": len(files), "input_bytes": int(sum(len(b) for b in files)), "gpu_call_median_ms": float(np.median(ms)),
             "gpu_call_max_ms": float(np.max(ms)), "cv2_imdecode_1_thread_ms": cv1, "cv2_imdecode_%d_threads_ms" % os.cpu_count(): cvn,
             "speedup_vs_cv2_1_thread": cv1 / float(np.median(ms)), "speedup_vs_cv2_all_threads": cvn / float(np.median(ms)),
             "host_parse_ms": parse, "call_stats": st}
        if not name.startswith("synthetic"):
            ctx.decode_images_orb(files, 1.0, 5000, images=False)
            fm = []
            for _ in range(max(3, a.reps // 2)):
                t0 = time.perf_counter(); ctx.decode_images_orb(files, 1.0, 5000, images=False); fm.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            imgs = [cv2.imdecode(b, cv2.IMREAD_COLOR) for b in bufs]
            for im in imgs:
                ctx.orb_detect_and_compute(im, 5000)
            chain = 1e3 * (time.perf_counter() - t0)
            r["fused_orb_call_median_ms"] = float(np.median(fm))
            r["cv2_imdecode_then_orb_detect_and_compute_ms"] = chain
        res[name] = r
    for name, files in loads.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ctx.decode_images(files)
        k = {p: 0.0 for p, _ in PHASES}; other = 0.0
        for e in prof.events():
            t = 1e-3 * e.device_time_total
            for p, keys in PHASES:
                if any(x in e.name for x in keys):
                    k[p] += t; break
            else:
                if "pg_" in e.name:
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
