"""SURVEY.md 8(f-1): the driver's glue (find2D3DMatches, mergeNewPointCloud) on the host and on the device.

Prints one JSON line per measurement:
  * host/sfm_glue.cpp against DeviceGlue on the test_glue --bench scene (24 views x 3000 features, 40k-point cloud, 8k new points)
    and on a 50-view scene (5000 features per view, 200k-point cloud, 20k new points), median of 5 after a warm-up; the device
    times include flattening the clouds, upload, download and applying the results (host/test_glue_device.cpp --bench);
  * the kernel split of one device find2D3DMatches and one mergeNewPointCloud on a scene of the 50-view size, from torch.profiler;
  * seconds["glue"] of the crazyhorse replay (runsfm.py) with the Python glue and with the device glue.
The card's name and power limit are printed with the numbers.  Usage: python tools/bench_glue.py
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, pl = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return {"card": name, "power_limit": pl}


def host_vs_device():
    exe = os.path.join(ROOT, "sfm-toy-library_b200", "host", "build", "test_glue_device")
    r = subprocess.run([exe, "1", "--bench"], capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        raise RuntimeError(r.stdout[-3000:] + r.stderr[-2000:])
    return [json.loads(l) for l in r.stdout.splitlines() if l.startswith("{")]


def kernel_split(ctx, V=50, F=5000, n_recon=200000, n_new=20000, seed=3):
    """Per-kernel device time of one find_2d3d_matches and one merge_point_cloud call (flat arrays, no Python containers)."""
    import torch
    from sfm_toy_library_b200 import capi
    rs = np.random.RandomState(seed)
    pairs, q, t, d, off = [], [], [], [], [0]
    for i in range(V):
        for j in range(i + 1, V):
            qq = np.nonzero(rs.rand(F) < 1 / 3)[0]
            pairs.append((i, j)); q.append(qq); t.append(rs.randint(0, F, len(qq))); d.append(rs.randint(0, 61, len(qq)).astype(np.float32))
            off.append(off[-1] + len(qq))
    index = ctx.match_index([F] * V, pairs, np.concatenate(q), np.concatenate(t), np.concatenate(d), off)

    def cloud(n, centres=None):
        k = rs.randint(2, 5, n)
        voff = np.zeros(n + 1, np.int32); voff[1:] = np.cumsum(k)
        views = np.argsort(rs.rand(n, V), axis=1)[:, :4]                              # 4 distinct views per point ...
        keep = np.arange(4)[None, :] < k[:, None]                                     # ... of which the first k, ascending
        img = np.sort(np.where(keep, views, V), axis=1)[keep].astype(np.int32)
        feat = rs.randint(0, F, voff[-1]).astype(np.int32)
        X = rs.uniform([-1, -1, 4], [1, 1, 6], (n, 3)) if centres is None else centres + rs.uniform(-0.012, 0.012, (n, 3))
        return X.astype(np.float32), (voff, img, feat)
    Xe, ev = cloud(n_recon)
    Xn, nv = cloud(n_new, Xe[rs.randint(0, n_recon, n_new)])
    done = (rs.rand(V) < 0.5).astype(np.uint8)
    for _ in range(2):
        index.find_2d3d_matches(done, *ev); index.merge_point_cloud(Xe, ev, Xn, nv)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter(); hits = index.find_2d3d_matches(done, *ev)[0]; t1 = time.perf_counter()
        r = index.merge_point_cloud(Xe, ev, Xn, nv); t2 = time.perf_counter()
    split = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA and "kernel" in e.key:
            split[e.key] = round(e.device_time_total / 1000.0, 4)
    index.close()
    return {"measurement": "kernel split (torch.profiler, one call each)", "views": V, "features_per_view": F, "cloud_points": n_recon,
            "new_points": n_new, "find2D3DMatches_call_ms": round(1e3 * (t1 - t0), 3), "mergeNewPointCloud_call_ms": round(1e3 * (t2 - t1), 3),
            "hits": int(len(hits)), "merge_counts": [int(x) for x in r["counts"]], "kernel_ms": split}


def crazyhorse(ctx, reps=2):
    from cfg1_util import Cfg1
    from sfm_toy_library_b200 import runsfm, stages
    cfg1 = Cfg1()
    common = dict(matchAllPairs=lambda feats, pairs: stages.matchAllPairs(feats, pairs, ctx=ctx),
                  triangulateViews=lambda *a: stages.triangulateViews(*a, ctx=ctx), adjustBundle=lambda *a: stages.adjustBundle(*a, ctx=ctx))
    device = dict(find2D3DMatches=lambda *a: stages.find2D3DMatches(*a, ctx=ctx),
                  mergeNewPointCloud=lambda *a: stages.mergeNewPointCloud(*a, ctx=ctx))
    out = {"measurement": "crazyhorse replay, seconds[\"glue\"] (best of %d)" % reps}
    for name, hooks in (("python_glue", {}), ("device_glue", device)):
        runs = []
        for _ in range(reps):
            sfm = runsfm.SfM(cfg1.features, cfg1.size, **common, **hooks)
            t0 = time.perf_counter(); sfm.runSfM(); wall = time.perf_counter() - t0
            runs.append((sfm.seconds["glue"], sfm.calls["glue"], wall, len(sfm.mReconstructionCloud)))
        best = min(runs)
        out[name] = {"glue_s": round(best[0], 4), "glue_calls": best[1], "wall_s": round(best[2], 3), "cloud": best[3]}
    return out


def main():
    from sfm_toy_library_b200 import capi
    info = card()
    for line in host_vs_device():
        print(json.dumps({**line, **info}))
    ctx = capi.Context(0)
    print(json.dumps({**kernel_split(ctx), **info}))
    print(json.dumps({**crazyhorse(ctx), **info}))
    ctx.close()


if __name__ == "__main__":
    main()
