"""BASELINE configs[0] (crazyhorse, 7 images) stage timing: the runSfM replay (sfm-toy-library_b200/runsfm.py) with the three
hot-path stages on the GPU through the drop-in call shape, beside the same replay on the CPU (cv2 for matching and
triangulation = the reference's own OpenCV calls, the oracle's Ceres restatement for adjustBundle).  RANSAC stages are
cv2 in both arms (SURVEY.md 8 f-2); the gpu_batched_essential arm also runs findCameraMatricesFromMatch on the device
(sfmb200_find_camera_matrices), the gpu_batched_essential_pairs arm the same stage for all pairs of a driver loop in one device
call (sfmb200_find_camera_matrices_pairs), the gpu_batched_homography arm the homography inliers of all pairs in one device call
(sfmb200_find_homography_pairs).  The triangulate_s line compares, alternated in the same run, the gpu_batched_essential_pairs
driver (one triangulateViews call per pair) with the gpu_batched_triangulate_pairs driver, which also triangulates all pairs of
an added view in one device call (sfmb200_triangulate_pairs).  Input: tests/golden/cfg1_crazyhorse.npz (pre-extracted ORB features).

    python tools/bench_cfg1.py [--reps 3] [--out gpurun_out/cfg1.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402


def run_arm(cfg1, arm, ctx=None, batched=True, threads=None, essential=False, homography=False, essential_pairs=False,
            triangulate_pairs=False):
    from sfm_toy_library_b200 import ransac, runsfm, stages
    kw = {}
    if arm == "gpu":
        kw = dict(matchFeatures=lambda a, b: stages.matchFeatures(a, b, ctx=ctx),
                  triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx),
                  adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx))
        if batched:
            kw["matchAllPairs"] = lambda feats, pairs: stages.matchAllPairs(feats, pairs, ctx=ctx)
        if essential:
            kw["findCameraMatricesFromMatch"] = lambda *a: ransac.findCameraMatricesFromMatch_gpu(*a, ctx=ctx)
        if essential_pairs:
            kw["findCameraMatricesManyPairs"] = lambda intr, f, pr, m: ransac.cameraMatricesManyPairs(intr, f, pr, m, ctx=ctx)
        if triangulate_pairs:
            kw["triangulateManyPairs"] = lambda *a: stages.triangulateManyPairs(*a, ctx=ctx)
        if homography:
            kw["homographyInliersAllPairs"] = lambda f, pr, m: ransac.homographyInliersAllPairs(f, pr, m, ctx=ctx)
    else:
        import cv2
        from oracle import cv2_stages
        if threads:
            cv2.setNumThreads(threads)
        kw = dict(matchFeatures=cv2_stages.matchFeatures, triangulateViews=cv2_stages.triangulateViews,
                  adjustBundle=lambda *a: cv2_stages.adjustBundle(*a, num_threads=1))     # the reference leaves Ceres at 1 thread
    feats = [type(f)(points=f.points.copy(), descriptors=f.descriptors.copy()) for f in cfg1.features]
    sfm = runsfm.SfM(feats, cfg1.size, **kw)
    t0 = time.perf_counter()
    sfm.runSfM()
    wall = time.perf_counter() - t0
    return {"wall_s": wall, "seconds": dict(sfm.seconds), "calls": dict(sfm.calls), "cloud": len(sfm.mReconstructionCloud),
            "hot_path_s": sfm.seconds["match"] + sfm.seconds["triangulate"] + sfm.seconds["bundle"]}


def measure_triangulate(cfg1, ctx, reps=3):
    """seconds["triangulate"] of the driver with the batched essential stage, triangulating pair by pair against one
    triangulateManyPairs call per added view; the two drivers alternate, the best of reps of each is kept"""
    from bench_stages import card
    arms = {"gpu_batched_essential_pairs": dict(essential_pairs=True), "gpu_batched_triangulate_pairs": dict(essential_pairs=True, triangulate_pairs=True)}
    runs = {k: [] for k in arms}
    for kw in arms.values():
        run_arm(cfg1, "gpu", ctx, **kw)
    for _ in range(reps):
        for k, kw in arms.items():
            runs[k].append(run_arm(cfg1, "gpu", ctx, **kw))
    best = {k: min(r, key=lambda x: x["seconds"]["triangulate"]) for k, r in runs.items()}
    name, pl = card()
    return {"card": name, "power_limit": pl, **{k: {"seconds": b["seconds"]["triangulate"], "calls": b["calls"]["triangulate"],
                                                    "all_runs_s": [x["seconds"]["triangulate"] for x in runs[k]]} for k, b in best.items()}}


def measure(reps=3):
    from cfg1_util import Cfg1
    from sfm_toy_library_b200 import capi
    cfg1 = Cfg1()
    ctx = capi.Context(0)
    out = {"workload": "crazyhorse 7 images x ORB(5000), runSfM replay (21 pairs, 21 triangulations, 6 bundle adjustments)"}
    run_arm(cfg1, "gpu", ctx)                                        # warm-up (allocations, module load)
    for name, kw in (("gpu_batched", dict(batched=True)), ("gpu_per_call", dict(batched=False))):
        runs = [run_arm(cfg1, "gpu", ctx, **kw) for _ in range(reps)]
        out[name] = min(runs, key=lambda r: r["hot_path_s"])
    run_arm(cfg1, "gpu", ctx, essential=True)
    runs = [run_arm(cfg1, "gpu", ctx, essential=True) for _ in range(reps)]
    out["gpu_batched_essential"] = min(runs, key=lambda r: r["seconds"]["essential"])
    run_arm(cfg1, "gpu", ctx, essential_pairs=True)
    runs = [run_arm(cfg1, "gpu", ctx, essential_pairs=True) for _ in range(reps)]
    out["gpu_batched_essential_pairs"] = min(runs, key=lambda r: r["seconds"]["essential"])
    out["essential_s"] = {k: out[k]["seconds"]["essential"] for k in ("gpu_batched", "gpu_batched_essential", "gpu_batched_essential_pairs")}
    out["triangulate_s"] = measure_triangulate(cfg1, ctx, reps)
    run_arm(cfg1, "gpu", ctx, homography=True)
    runs = [run_arm(cfg1, "gpu", ctx, homography=True) for _ in range(reps)]
    out["gpu_batched_homography"] = min(runs, key=lambda r: r["seconds"]["homography"])
    out["homography_s"] = {"gpu_batched": out["gpu_batched"]["seconds"]["homography"],
                           "gpu_batched_homography": out["gpu_batched_homography"]["seconds"]["homography"]}
    os.environ["SFMB200_MATCH_CACHE"] = "0"
    runs = [run_arm(cfg1, "gpu", ctx, batched=False) for _ in range(reps)]
    out["gpu_per_call_nocache"] = min(runs, key=lambda r: r["hot_path_s"])
    del os.environ["SFMB200_MATCH_CACHE"]
    ncpu = os.cpu_count() or 1
    out["cpu_cv2_all_threads"] = min((run_arm(cfg1, "cpu", threads=ncpu) for _ in range(max(1, reps - 1))), key=lambda r: r["hot_path_s"])
    if reps >= 3:
        out["cpu_cv2_1_thread"] = run_arm(cfg1, "cpu", threads=1)
    out["cpu_threads"] = ncpu
    g, c = out["gpu_batched"], out["cpu_cv2_all_threads"]
    out["speedup_hot_path"] = c["hot_path_s"] / g["hot_path_s"]
    out["speedup_per_stage"] = {k: c["seconds"][k] / max(g["seconds"][k], 1e-9) for k in ("match", "triangulate", "bundle")}
    ctx.close()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    r = measure(a.reps)
    txt = json.dumps(r, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        open(a.out, "w").write(txt)
