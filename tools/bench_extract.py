"""tools/bench_extract.py -- the feature front end from JPEG files: sfmb200_decode_jpeg_extract_orb (decode, downscale and ORB with the
images staying on the device) against the two-call chain it replaces (decode_jpeg[_scaled], which downloads the images, then one
orb_detect_and_compute batch per image size, which uploads them again).  Workloads:
    crazyhorse x7, crazyhorse x50                       (1024 x 768 photographs, -s 1)
    50 synthetic 4032 x 3024 files, every other one with EXIF orientation 6 (decodes to 3024 x 4032), at -s 1 and 0.5
Each line: ms per image of the fused call with and without the image download and of the chain, and the bytes that crossed PCIe
(uploads of the files and images, downloads of the images; key points and descriptors, equal for all, are not counted).  The card's name
and power limit are read in the same run.  Results are checked equal before timing.
    python tools/bench_extract.py [--reps 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import jpeg_util as J  # noqa: E402
from sfm_toy_library_b200 import capi  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi: %s)" % r.stderr.strip()


def chain(ctx, blobs, scale):
    imgs = ctx.decode_jpeg(blobs, scale)
    st = ctx.jpeg_last_stats()
    by_shape = {}
    for i, im in enumerate(imgs):
        by_shape.setdefault(im.shape, []).append(i)
    feats = [None] * len(imgs)
    for idx in by_shape.values():
        for i, f in zip(idx, ctx.orb_detect_and_compute([imgs[i] for i in idx], 5000)):
            feats[i] = f
    pcie = st["upload_bytes"] + st["download_bytes"] + sum(im.nbytes for im in imgs)
    return imgs, feats, pcie


def fused(ctx, blobs, scale, images):
    imgs, feats = ctx.decode_jpeg_orb(blobs, scale, images=images)
    st = ctx.jpeg_last_stats()
    return imgs, feats, st["upload_bytes"] + st["download_bytes"]


def timed(fn, reps):
    fn()                                                  # warm-up: allocations at this size
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); out = fn(); ts.append(time.perf_counter() - t)
    return min(ts), sorted(ts)[len(ts) // 2], out


def run(name, blobs, scale, reps, ctx):
    n = len(blobs)
    _, fa, _ = fused(ctx, blobs, scale, True)
    _, fb, _ = chain(ctx, blobs, scale)
    same = all(a[0].shape == b[0].shape and (a[0] == b[0]).all() and (a[1] == b[1]).all() for a, b in zip(fa, fb))
    line = {"workload": name, "images": n, "scale": scale, "equal_results": bool(same)}
    for key, fn in (("chain", lambda: chain(ctx, blobs, scale)), ("fused_with_images", lambda: fused(ctx, blobs, scale, True)),
                    ("fused_no_images", lambda: fused(ctx, blobs, scale, False))):
        best, med, out = timed(fn, reps)
        line[key] = {"ms_per_image_best": round(best * 1e3 / n, 3), "ms_per_image_median": round(med * 1e3 / n, 3),
                     "pcie_bytes": int(out[2])}
    line["speedup_no_images_vs_chain"] = round(line["chain"]["ms_per_image_best"] / line["fused_no_images"]["ms_per_image_best"], 3)
    line["speedup_with_images_vs_chain"] = round(line["chain"]["ms_per_image_best"] / line["fused_with_images"]["ms_per_image_best"], 3)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5); ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = capi.Context(0)
    lines = [{"card": card(), "note": "name, power limit, max SM clock, read in this run"}]
    horse = J.crazyhorse()
    big = [J.encode(4032, 3024, seed=s) for s in (1, 2)]
    big_rot = [b[:2] + J.exif_app1(6) + b[2:] for b in big]
    phone = [(big if k % 2 == 0 else big_rot)[(k // 2) % 2] for k in range(50)]
    for name, blobs, scale in (("crazyhorse_x7", [horse] * 7, 1.0), ("crazyhorse_x50", [horse] * 50, 1.0),
                               ("phone_4032x3024_x50_half_rotated", phone, 1.0), ("phone_4032x3024_x50_half_rotated", phone, 0.5)):
        lines.append(run(name, blobs, scale, a.reps, ctx))
        print(json.dumps(lines[-1]), flush=True)
    ctx.close()
    print(json.dumps(lines[0]))
    if a.out:
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
