#!/usr/bin/env python
"""Secondary metrics of SURVEY.md section 8(d): all-pairs matching (BASELINE.json config 4, reference-faithful Hamming)
and batched triangulation (config 5), each with resident-input device timing (CUDA events on the library stream),
the host-buffer C-ABI call, a roofline object and a CPU baseline (cv2 = the OpenCV code the reference calls).
Prints one JSON line per stage.  Usage: python tools/bench_stages.py [--images 50] [--features 5000] [--points 1000000]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        return float(json.load(open(p))["hbm_gbs"]), "measured"
    except Exception:
        return 3350.0, "H100 SXM data sheet HBM3 (not measured)"


def tensor_peak_tops():
    """int8 dense rate = 2x the bf16 dense rate; bf16 is the measured cuBLAS figure of MEASURED_PEAKS.json (burst)."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        return 2.0 * float(json.load(open(p))["bf16_tflops"]), "2 x measured bf16 (MEASURED_PEAKS.json bf16_tflops)"
    except Exception:
        return 1979.0, "H100 SXM data sheet dense int8 (not measured)"


def _timed(ctx, stream, flush, fn, reps):
    import torch
    ts = []
    for _ in range(reps + 1):
        with torch.cuda.stream(stream):
            flush.zero_()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        ctx.synchronize(); e0.record(stream); fn(); e1.record(stream); ctx.synchronize(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.mean(ts[1:]))


def measure_match(ctx, stream, flush, images=50, features=5000, reps=5, norm="hamming"):
    """BASELINE configs[3]: all-pairs matching of `images` x `features` descriptors.  norm="hamming": the reference-faithful case
    (ORB-256, SfM2DFeatureUtilities.cpp:53-71); norm="l2": the BASELINE wording (SIFT-128, cv::BFMatcher(NORM_L2)), exact u8 GEMM."""
    import torch
    from sfm_toy_library_b200 import capi, synth
    if norm == "hamming":
        descs = synth.make_descriptor_set(images, n=features); kbits = 256
    else:
        descs = [synth.make_sift_like(0, features)]
        for i in range(1, images):
            descs.append(synth.make_sift_like(i, features, prev=descs[-1]))
        kbits = 128
    pairs = [(i, j) for i in range(images) for j in range(i + 1, images)]
    ds = ctx.descriptor_set(descs, norm=norm)
    rows = features * len(pairs)
    dq = torch.empty(rows, dtype=torch.int32, device="cuda"); dt_ = torch.empty(rows, dtype=torch.int32, device="cuda")
    dd = torch.empty(rows, dtype=torch.float32, device="cuda"); dst = torch.empty(len(pairs) + 1, dtype=torch.int32, device="cuda")
    dtot = torch.empty(1, dtype=torch.int64, device="cuda")
    l0 = ctx.kernel_launches
    ms = _timed(ctx, stream, flush, lambda: ds.match_pairs_device(pairs, dq.data_ptr(), dt_.data_ptr(), dd.data_ptr(), dst.data_ptr(), dtot.data_ptr()), reps)
    launches = (ctx.kernel_launches - l0) // (reps + 1)
    assert int(dtot.item()) >= 0, "tensor-core pipeline error flag"
    ds.match_pairs(pairs)                                   # untimed: first call allocates the pinned result staging
    t0 = time.perf_counter(); res = ds.match_pairs(pairs); resident_s = time.perf_counter() - t0
    ds.close()
    # true end-to-end through the batched C-ABI calls with HOST buffers: descriptor upload + expansion (descset_create),
    # all pairs, survivors read back, set destroyed -- what a host that holds cv::Mat descriptors pays
    e2e = []
    packed = np.ascontiguousarray(np.concatenate(descs, 0)); sizes = [len(d) for d in descs]     # the host's descriptor rows, as a C++ caller holds them
    bufs = None
    for _ in range(4):                                      # the three C calls alone: result buffers are the caller's (allocated and touched once)
        t0 = time.perf_counter()
        d2 = capi.DescriptorSet.from_packed(ctx, packed, sizes, norm=norm)
        call, bufs = d2.match_pairs_prepare(pairs, buffers=bufs)
        off2, cnt2 = call()
        d2.close()
        t3 = time.perf_counter()
        e2e.append(t3 - t0)
    e2e_s = min(e2e[1:])
    assert int(cnt2.sum()) == int(sum(len(r[0]) for r in res))
    n_matches = int(sum(len(r[0]) for r in res))
    h2d = int(sum(d.nbytes for d in descs)); d2h = 12 * n_matches + 4 * len(pairs)
    dist_evals = float(features) ** 2 * len(pairs)
    import cv2
    cpu = {}
    for thr in (1, os.cpu_count() or 1):
        cv2.setNumThreads(thr)
        m = cv2.DescriptorMatcher_create("BruteForce-Hamming" if norm == "hamming" else "BruteForce")
        npairs_cpu = 2 if thr == 1 else 8
        t0 = time.perf_counter()
        for (i, j) in pairs[:npairs_cpu]:
            m.knnMatch(descs[i], descs[j], 2)
        cpu[thr] = npairs_cpu / (time.perf_counter() - t0)
    peak, peak_src = tensor_peak_tops()
    ach = 2 * dist_evals * kbits / (ms * 1e-3) / 1e12
    what = "5000x5000 ORB-256 Hamming" if norm == "hamming" else "5000x5000 SIFT-128 L2"
    return {"stage": "match_" + norm, "metric": f"image pairs matched per second ({what}, knn2 + ratio)", "value": len(pairs) / (ms * 1e-3),
            "unit": "pairs/s", "ms_per_step": ms, "pairs": len(pairs), "features": features, "matches": n_matches, "dtype": "s8 x s8 -> s32" if norm == "hamming" else "u8 x u8 -> s32",
            "descriptor_pairs_per_s": dist_evals / (ms * 1e-3), "gpu_launches": int(launches),
            "e2e": {"value": len(pairs) / e2e_s, "unit": "pairs/s", "seconds": e2e_s, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                    "note": "sfmb200_descset_create (upload + operand expansion) + sfmb200_match_pairs (caller-owned host result buffers) + destroy; the first repetition (buffer allocation) is dropped",
                    "resident_descriptors_pairs_per_s": len(pairs) / resident_s},
            "roofline": {"bound": "tensor", "achieved": ach, "peak": peak, "unit": "TOP/s", "frac": ach / peak, "peak_source": peak_src,
                         "kernel": "knn2_tc_kernel<L2=%s> (wgmma m64n128k32 s8/u8)" % ("true" if norm != "hamming" else "false"),
                         "note": f"exact integer GEMM form: 2*Nq*Nt*{kbits} ops per pair; descriptor bytes are negligible (L2-resident)"},
            "cpu_baseline": {"value": cpu[max(cpu)], "unit": "pairs/s", "cores": max(cpu), "kind": "reference", "single_thread_pairs_per_s": cpu[1],
                             "sample": "cv2 BruteForce knnMatch(k=2) on the first pairs of the same set"}}


def measure_triangulate(ctx, stream, flush, points=1_000_000, reps=5):
    """BASELINE configs[4]: triangulateViews on `points` matches in one call."""
    import cv2
    import torch
    from sfm_toy_library_b200 import synth
    hbm, src = peaks()
    p = synth.make_triangulation_problem(points, seed=0)
    m = points
    dl = torch.from_numpy(p["ptsL"]).cuda(); dr = torch.from_numpy(p["ptsR"]).cuda()
    dX = torch.empty(m * 3, dtype=torch.float32, device="cuda"); dk = torch.empty(m, dtype=torch.uint8, device="cuda"); dn = torch.empty(1, dtype=torch.int32, device="cuda")
    ms = _timed(ctx, stream, flush, lambda: ctx.triangulate_device(p["K"], p["Pl"], p["Pr"], dl.data_ptr(), dr.data_ptr(), None, None, m, dX.data_ptr(), dk.data_ptr(), dn.data_ptr()), reps)
    ctx.triangulate(p["K"], p["Pl"], p["Pr"], p["ptsL"], p["ptsR"])      # untimed: first call grows the device scratch
    t0 = time.perf_counter(); X, keep, nk = ctx.triangulate(p["K"], p["Pl"], p["Pr"], p["ptsL"], p["ptsR"]); e2e_s = time.perf_counter() - t0
    from oracle import cv2_reference as ref
    cv2.setNumThreads(os.cpu_count() or 1)
    ns = min(m, 100_000)
    t0 = time.perf_counter(); ref.triangulate_views(p["K"], p["Pl"], p["Pr"], p["ptsL"][:ns], p["ptsR"][:ns]); cpu_s = time.perf_counter() - t0
    abytes = 29 * m
    return {"stage": "triangulate", "metric": "point pairs triangulated per second (DLT + reprojection filter)", "value": m / (ms * 1e-3), "unit": "points/s",
            "ms_per_step": ms, "points": m, "kept": int(nk), "dtype": "f64 inside, f32 in/out", "gpu_launches": 1,
            "e2e": {"value": m / e2e_s, "unit": "points/s", "h2d_bytes_per_step": 16 * m, "d2h_bytes_per_step": 13 * m, "note": "sfmb200_triangulate with host buffers"},
            "roofline": {"bound": "hbm", "achieved": abytes / (ms * 1e-3) / 1e9, "peak": hbm, "unit": "GB/s", "frac": abytes / (ms * 1e-3) / 1e9 / hbm,
                         "peak_source": src, "algorithmic_bytes": abytes, "note": "fp64 ALU bound in practice (closed-form smallest eigenvector, Jacobi SVD fallback)"},
            "cpu_baseline": {"value": ns / cpu_s, "unit": "points/s", "cores": 1, "kind": "reference",
                             "sample": f"cv2 replay of triangulateViews on the first {ns} points (cv::triangulatePoints is serial)"}}


def card():
    """name and power limit of the card the numbers were measured on"""
    import subprocess
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


ESSENTIAL_KERNELS = ("essential_cv_sample_kernel", "essential_solve_kernel", "essential_score_kernel", "essential_select_kernel", "essential_cheirality_kernel",
                     "essential_pose_kernel")


def synthetic_essential_set(images=50, seed=0):
    """Seeded all-pairs set: per pair a two-view scene (tests/essential_util.synthetic_scene) of 200-1200 matches at 30-70 %
    outliers and 0.5 px noise, its points appended to the two images."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from essential_util import synthetic_scene
    rs = np.random.RandomState(seed)
    pts = [[] for _ in range(images)]; sizes = [0] * images
    pairs, mq, mt, off = [], [], [], [0]
    for i in range(images):
        for j in range(i + 1, images):
            n = int(rs.randint(200, 1201)); r = rs.uniform(0.3, 0.7)
            a, b, *_ = synthetic_scene(int(rs.randint(1 << 30)), n, noise_px=0.5, outliers=r)
            pts[i].append(a); pts[j].append(b)
            mq.append(np.arange(n, dtype=np.int32) + sizes[i]); mt.append(np.arange(n, dtype=np.int32) + sizes[j])
            sizes[i] += n; sizes[j] += n
            pairs.append((i, j)); off.append(off[-1] + n)
    return [np.concatenate(p) for p in pts], np.array(pairs, np.int32), np.concatenate(mq), np.concatenate(mt), np.array(off, np.int64)


def essential_kernel_ms(fn):
    """device time per K5 kernel (ms, summed over its launches) of one fn() under torch.profiler"""
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in ESSENTIAL_KERNELS}
    for e in prof.events():
        for k in ESSENTIAL_KERNELS:
            if k in e.name:
                out[k] += 1e-3 * e.device_time_total
    out["total"] = sum(out.values())
    return out


def measure_essential(ctx, reps=20, profile=False):
    """findCameraMatricesFromMatch (SfMStereoUtilities.cpp:74-118) on the 21 crazyhorse pairs of tests/golden/cfg1_crazyhorse.npz:
    sfmb200_find_camera_matrices (host clock around the synchronised call, warmed up, median over reps per pair) against
    cv2.findEssentialMat(RANSAC, 0.999, 1 px) + cv2.recoverPose on one thread and on all threads.  Then, in the same run, the 21
    pairs as 21 single calls and in one sfmb200_find_camera_matrices_pairs call (host clock, median over reps), a seeded synthetic
    50-image set (1225 pairs) in one call, and with profile=True the per-kernel device time of each from torch.profiler in a
    separate pass.  Last, the two samplers alternated round by round (seeded against OpenCV's samples, sfmb200_essential_options.sampler)
    on the same three workloads, and their kernel split."""
    import cv2
    from sfm_toy_library_b200 import capi
    g = np.load(os.path.join(ROOT, "tests", "golden", "cfg1_crazyhorse.npz"))
    K = np.array([[2500, 0, 512], [0, 2500, 384], [0, 0, 1]], np.float32)
    pairs = []
    for p, (i, j) in enumerate(g["pairs"]):
        a = g[f"pts_{int(i)}"][g[f"match_{p}_q"]]; b = g[f"pts_{int(j)}"][g[f"match_{p}_t"]]
        pairs.append((np.ascontiguousarray(a), np.ascontiguousarray(b)))
    gpu = []
    for a, b in pairs:
        ctx.find_camera_matrices(K, a, b)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); ctx.find_camera_matrices(K, a, b); ts.append(time.perf_counter() - t0)
        gpu.append(1e3 * float(np.median(ts)))

    def cv_ms(threads):
        cv2.setNumThreads(threads)
        out = []
        for a, b in pairs:
            t0 = time.perf_counter()
            E, m = cv2.findEssentialMat(a, b, 2500.0, (512.0, 384.0), cv2.RANSAC, 0.999, 1.0)
            cv2.recoverPose(E[:3], a, b, focal=2500.0, pp=(512.0, 384.0), mask=m)
            out.append(1e3 * (time.perf_counter() - t0))
        return out
    one = cv_ms(1); allt = cv_ms(os.cpu_count() or 1)
    cv2.setNumThreads(-1)

    feats = [g[f"pts_{i}"] for i in range(len(g["files"]))]
    ch_pairs = np.array(g["pairs"], np.int32)
    ch_q, ch_t, ch_off = capi.flatten_matches([g[f"match_{p}_q"] for p in range(len(ch_pairs))], [g[f"match_{p}_t"] for p in range(len(ch_pairs))])
    sy = synthetic_essential_set()

    def timed(fn, n):
        fn()
        ts = []
        for _ in range(n):
            t0 = time.perf_counter(); fn(); ts.append(1e3 * (time.perf_counter() - t0))
        return ts
    singles = lambda: [ctx.find_camera_matrices(K, a, b) for a, b in pairs]
    batched = lambda: ctx.find_camera_matrices_pairs(K, feats, ch_pairs, ch_q, ch_t, ch_off)
    synthetic = lambda: ctx.find_camera_matrices_pairs(K, *sy)
    t_single, t_batch = [], []
    for _ in range(reps // 2):                   # alternated, so both see the same state of the shared machine
        t_single += timed(singles, 1); t_batch += timed(batched, 1)
    t_syn = timed(synthetic, 5)
    kernels = {"crazyhorse_21_single_calls": essential_kernel_ms(singles), "crazyhorse_21_one_call": essential_kernel_ms(batched),
               "synthetic_1225_one_call": essential_kernel_ms(synthetic)} if profile else "not profiled"
    samplers = measure_essential_samplers(ctx, K, pairs, (feats, ch_pairs, ch_q, ch_t, ch_off), sy, reps, profile)
    name, pl = card()
    return {"metric": "essential_ransac_pose_ms_per_call", "gpu_median_ms": float(np.median(gpu)), "gpu_max_ms": float(np.max(gpu)),
            "cv2_1thread_median_ms": float(np.median(one)), "cv2_all_threads_median_ms": float(np.median(allt)),
            "speedup_vs_cv2_1thread": float(np.median(one) / np.median(gpu)), "pairs": len(pairs), "matches": [int(len(a)) for a, _ in pairs],
            "card": name, "power_limit": pl, "cpu_threads": os.cpu_count(),
            "crazyhorse_21_single_calls_median_ms": float(np.median(t_single)), "crazyhorse_21_one_call_median_ms": float(np.median(t_batch)),
            "crazyhorse_21_speedup_one_call": float(np.median(t_single) / np.median(t_batch)),
            "synthetic_1225_one_call_median_ms": float(np.median(t_syn)), "synthetic_1225_one_call_max_ms": float(np.max(t_syn)),
            "synthetic_matches": int(sy[4][-1]), "kernel_ms_torch_profiler": kernels, "samplers": samplers,
            "detail": {"gpu_ms": gpu, "cv2_1thread_ms": one, "cv2_all_threads_ms": allt, "crazyhorse_21_single_calls_ms": t_single,
                       "crazyhorse_21_one_call_ms": t_batch, "synthetic_1225_one_call_ms": t_syn}}


def measure_essential_samplers(ctx, K, pairs, crazyhorse, synthetic, reps, profile):
    """The seeded arm (the default sampler) against the opencv arm (cv::findEssentialMat's own samples) in alternating rounds:
    crazyhorse per call (median over rounds per pair, then over pairs), the 21 pairs in one call, the 1225 synthetic pairs in one call
    (host clock around synchronised calls, every call warmed up before the rounds); with profile=True each arm's kernel split."""
    from sfm_toy_library_b200 import capi
    arms = {"seeded": {}, "opencv": {"sampler": capi.SAMPLER_OPENCV}}
    work = {"crazyhorse_21_one_call": lambda kw: ctx.find_camera_matrices_pairs(K, *crazyhorse, **kw),
            "synthetic_1225_one_call": lambda kw: ctx.find_camera_matrices_pairs(K, *synthetic, **kw)}
    per_pair = {k: [[] for _ in pairs] for k in arms}
    calls = {k: {w: [] for w in work} for k in arms}
    for kw in arms.values():                      # warm-up of every shape in both arms
        for a, b in pairs:
            ctx.find_camera_matrices(K, a, b, **kw)
        for fn in work.values():
            fn(kw)

    def clock(fn):
        t0 = time.perf_counter(); fn(); return 1e3 * (time.perf_counter() - t0)
    for _ in range(max(reps // 2, 1)):
        for k, kw in arms.items():
            for p, (a, b) in enumerate(pairs):
                per_pair[k][p].append(clock(lambda: ctx.find_camera_matrices(K, a, b, **kw)))
            for w, fn in work.items():
                calls[k][w].append(clock(lambda: fn(kw)))
    out = {}
    for k, kw in arms.items():
        out[k] = {"crazyhorse_per_call_median_ms": float(np.median([np.median(x) for x in per_pair[k]])),
                  "crazyhorse_per_call_max_ms": float(np.max([np.median(x) for x in per_pair[k]]))}
        for w in work:
            out[k][w + "_median_ms"] = float(np.median(calls[k][w])); out[k][w + "_ms"] = calls[k][w]
        if profile:
            out[k]["kernel_ms_torch_profiler"] = {
                "crazyhorse_21_single_calls": essential_kernel_ms(lambda: [ctx.find_camera_matrices(K, a, b, **kw) for a, b in pairs]),
                **{w: essential_kernel_ms(lambda: fn(kw)) for w, fn in work.items()}}
    return out


def synthetic_homography_set(images=50, seed=0):
    """Seeded all-pairs set: per pair a planar scene of 200-1200 matches at 30-70 % outliers, its points appended to the two images."""
    rs = np.random.RandomState(seed)
    pts = [[] for _ in range(images)]; sizes = [0] * images
    pairs, mq, mt, off = [], [], [], [0]
    for i in range(images):
        for j in range(i + 1, images):
            n = int(rs.randint(200, 1201)); r = rs.uniform(0.3, 0.7)
            H = np.eye(3) + np.r_[rs.normal(0, 0.08, 6), rs.normal(0, 1e-4, 2), 0].reshape(3, 3)
            a = np.c_[rs.uniform(0, 1024, n), rs.uniform(0, 768, n)]
            ph = np.c_[a, np.ones(n)] @ H.T
            b = ph[:, :2] / ph[:, 2:] + rs.normal(0, 0.5, (n, 2))
            k = int(r * n); o = rs.choice(n, k, replace=False); b[o] = np.c_[rs.uniform(0, 1024, k), rs.uniform(0, 768, k)]
            pts[i].append(a.astype(np.float32)); pts[j].append(b.astype(np.float32))
            mq.append(np.arange(n, dtype=np.int32) + sizes[i]); mt.append(np.arange(n, dtype=np.int32) + sizes[j])
            sizes[i] += n; sizes[j] += n
            pairs.append((i, j)); off.append(off[-1] + n)
    return [np.concatenate(p) for p in pts], np.array(pairs, np.int32), np.concatenate(mq), np.concatenate(mt), np.array(off, np.int64)


def measure_homography(ctx, images=50, reps=3):
    """findHomographyInliers (SfMStereoUtilities.cpp:51-72): sfmb200_find_homography_pairs, host clock around the synchronised
    call (warmed up; median and max over reps), on the 21 crazyhorse pairs one call per pair and all in one call, and on a seeded
    synthetic 50-image set (1225 pairs) in one call; cv2.findHomography(RANSAC, 10) on one host thread for the same work; the
    kernel time of the batched calls from torch.profiler in a separate pass."""
    import cv2
    import torch
    from sfm_toy_library_b200 import capi
    g = np.load(os.path.join(ROOT, "tests", "golden", "cfg1_crazyhorse.npz"))
    feats = [g[f"pts_{i}"] for i in range(len(g["files"]))]
    ch_pairs = np.array(g["pairs"], np.int32)
    ch_q, ch_t, ch_off = capi.flatten_matches([g[f"match_{p}_q"] for p in range(len(ch_pairs))], [g[f"match_{p}_t"] for p in range(len(ch_pairs))])
    sy = synthetic_homography_set(images)

    def timed(fn):
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); fn(); ts.append(1e3 * (time.perf_counter() - t0))
        return ts
    per_pair = []
    for p in range(len(ch_pairs)):
        sl = slice(int(ch_off[p]), int(ch_off[p + 1]))
        per_pair.append(timed(lambda: ctx.find_homography_pairs(feats, ch_pairs[p:p + 1], ch_q[sl], ch_t[sl], np.array([0, sl.stop - sl.start]))))
    batched = timed(lambda: ctx.find_homography_pairs(feats, ch_pairs, ch_q, ch_t, ch_off))
    syn = timed(lambda: ctx.find_homography_pairs(*sy))

    def cv_ms(points, pairs, q, t, off):
        cv2.setNumThreads(1)
        t0 = time.perf_counter()
        for p, (i, j) in enumerate(pairs):
            sl = slice(int(off[p]), int(off[p + 1]))
            cv2.findHomography(points[i][q[sl]], points[j][t[sl]], cv2.RANSAC, 10.0)
        cv2.setNumThreads(-1)
        return 1e3 * (time.perf_counter() - t0)
    cv_ch = cv_ms(feats, ch_pairs, ch_q, ch_t, ch_off); cv_syn = cv_ms(*sy)
    kernel = {}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ctx.find_homography_pairs(feats, ch_pairs, ch_q, ch_t, ch_off)
        ctx.find_homography_pairs(*sy)
    for e in prof.events():
        if "homography_pairs_kernel" in e.name:
            kernel.setdefault("crazyhorse_21" if not kernel else "synthetic_1225", 1e-3 * e.device_time_total)
    name, pl = card()
    med = [float(np.median(x)) for x in per_pair]
    return {"metric": "homography_ransac_ms_per_call", "card": name, "power_limit": pl,
            "crazyhorse_per_pair_median_ms": float(np.median(med)), "crazyhorse_per_pair_max_ms": float(np.max([max(x) for x in per_pair])),
            "crazyhorse_per_pair_sum_of_medians_ms": float(np.sum(med)),
            "crazyhorse_21_one_call_median_ms": float(np.median(batched)), "crazyhorse_21_one_call_max_ms": float(np.max(batched)),
            "synthetic_1225_one_call_median_ms": float(np.median(syn)), "synthetic_1225_one_call_max_ms": float(np.max(syn)),
            "synthetic_matches": int(sy[4][-1]), "cv2_1thread_crazyhorse_21_ms": cv_ch, "cv2_1thread_synthetic_1225_ms": cv_syn,
            "kernel_ms_torch_profiler": kernel}


def measure_triangulate_pairs(ctx, reps=20, profile=False):
    """triangulateViews (SfMStereoUtilities.cpp:120-206) batched per driver loop: host clock around the synchronised call, warmed up,
    median and max over reps, the two arms alternated in the same run.
      - the 20 addMoreViewsToReconstruction triangulations of tests/golden/cfg1_crazyhorse.npz (every recorded call after the
        baseline's): 20 sfmb200_triangulate calls against one sfmb200_triangulate_pairs call per added view (5 calls);
      - synth.make_triangulation_pairs(50): 1225 single calls against one call.
    With profile=True, the device time of triangulate_kernel / triangulate_pairs_kernel of each arm from torch.profiler in a
    separate pass."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from cfg1_util import Cfg1
    from sfm_toy_library_b200 import capi, synth
    cfg1 = Cfg1()
    pts = [f.points for f in cfg1.features]
    loops = {}
    for k in range(1, cfg1.n_tri):
        loops.setdefault(cfg1.tri(k)["K"].tobytes(), []).append(cfg1.tri(k))
    loops = list(loops.values())
    ch_single = [(c["K"], c["Pl"], c["Pr"], pts[int(c["pair"][0])], pts[int(c["pair"][1])], c["mq"], c["mt"]) for lp in loops for c in lp]
    ch_batch = []
    for lp in loops:
        ch_batch.append((lp[0]["K"], [(c["Pl"], c["Pr"]) for c in lp], pts, [tuple(int(x) for x in c["pair"]) for c in lp],
                         *capi.flatten_matches([c["mq"] for c in lp], [c["mt"] for c in lp])))
    K, poses, spts, spairs, smq, smt, soff = sy = synth.make_triangulation_pairs(50, seed=0)
    sy_single = [(K, poses[p][0], poses[p][1], spts[i], spts[j], smq[soff[p]:soff[p + 1]], smt[soff[p]:soff[p + 1]]) for p, (i, j) in enumerate(spairs)]
    arms = {"crazyhorse_20_single_calls": lambda: [ctx.triangulate(*a) for a in ch_single],
            "crazyhorse_20_in_5_calls": lambda: [ctx.triangulate_pairs(*a) for a in ch_batch],
            "synthetic_1225_single_calls": lambda: [ctx.triangulate(*a) for a in sy_single],
            "synthetic_1225_one_call": lambda: ctx.triangulate_pairs(*sy)}
    per_call = []                                       # one single call at a time, per crazyhorse call
    for a in ch_single:
        ctx.triangulate(*a)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); ctx.triangulate(*a); ts.append(1e3 * (time.perf_counter() - t0))
        per_call.append(float(np.median(ts)))
    times = {k: [] for k in arms}
    for f in arms.values():
        f()
    for _ in range(reps):                               # alternated, so both arms see the same state of the shared machine
        for k, f in arms.items():
            t0 = time.perf_counter(); f(); times[k].append(1e3 * (time.perf_counter() - t0))
    kernels = "not profiled"
    if profile:
        import torch
        kernels = {}
        for k, f in arms.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                f()
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if "triangulate" in e.name and "kernel" in e.name]
            kernels[k] = {"ms": 1e-3 * sum(e.device_time_total for e in ev), "launches": len(ev)}
    name, pl = card()
    out = {"metric": "triangulate_pairs_ms", "card": name, "power_limit": pl, "reps": reps,
           "crazyhorse_matches_per_call": [int(len(a[5])) for a in ch_single], "crazyhorse_calls_per_added_view": [len(lp) for lp in loops],
           "crazyhorse_single_call_median_ms": float(np.median(per_call)), "crazyhorse_single_call_max_ms": float(np.max(per_call)),
           "synthetic_pairs": len(spairs), "synthetic_matches": int(soff[-1]), "kernel_ms_torch_profiler": kernels}
    for k, ts in times.items():
        out[k + "_median_ms"] = float(np.median(ts)); out[k + "_max_ms"] = float(np.max(ts))
    out["crazyhorse_speedup_batched"] = out["crazyhorse_20_single_calls_median_ms"] / out["crazyhorse_20_in_5_calls_median_ms"]
    out["synthetic_speedup_batched"] = out["synthetic_1225_single_calls_median_ms"] / out["synthetic_1225_one_call_median_ms"]
    return out


POSE_KERNELS = ("pose_solve_kernel", "pose_score_kernel", "pose_select_kernel", "pose_refit_kernel")


def pose_kernel_ms(fn):
    """device time per K9 kernel (ms, summed over its launches) of one fn() under torch.profiler"""
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in POSE_KERNELS}
    for e in prof.events():
        for k in POSE_KERNELS:
            if k in e.name:
                out[k] += 1e-3 * e.device_time_total
    out["total"] = sum(out.values())
    return out


def measure_pose(ctx, reps=20, profile=False):
    """findCameraPoseFrom2D3DMatch (SfMStereoUtilities.cpp:208-243) on the five PnP sets of the crazyhorse replay
    (tests/golden/cfg1_crazyhorse.npz, with the intrinsics of each call): sfmb200_find_camera_pose (host clock around the synchronised
    call, warmed up, median over reps per set) against cv2.solvePnPRansac(100, 10 px, 0.99) on one thread and on all threads; a
    seeded synthetic set of 100 000 correspondences with 30 % outliers; with profile=True the per-kernel device time from
    torch.profiler in a separate pass."""
    import cv2
    g = np.load(os.path.join(ROOT, "tests", "golden", "cfg1_crazyhorse.npz"))
    sets = [(g[f"pnp_{k}_p3"], g[f"pnp_{k}_p2"], np.asarray(g[f"ba_{k}_K_after"], np.float32)) for k in range(int(g["n_pnp"]))]
    rs = np.random.RandomState(0)
    n = 100_000
    Ks = np.array([[1200, 0, 640], [0, 1150, 360], [0, 0, 1]], np.float32)
    Xc = np.c_[rs.uniform(-3, 3, (n, 2)), rs.uniform(4, 12, n)]
    uv = Xc[:, :2] / Xc[:, 2:] * [1200, 1150] + [640, 360] + rs.normal(0, 0.5, (n, 2))
    bad = rs.uniform(size=n) < 0.3
    uv[bad] = rs.uniform([0, 0], [1280, 720], (int(bad.sum()), 2))
    syn = (Xc.astype(np.float32), uv.astype(np.float32), Ks)

    def timed(X, p2, K, r):
        ctx.find_camera_pose(K, X, p2)
        ts = []
        for _ in range(r):
            t0 = time.perf_counter(); ctx.find_camera_pose(K, X, p2); ts.append(1e3 * (time.perf_counter() - t0))
        return ts
    gpu = [float(np.median(timed(X, p2, K, reps))) for X, p2, K in sets]
    t_syn = timed(*syn, 5)

    def cv_ms(threads, data, r=5):
        cv2.setNumThreads(threads)
        out = []
        for X, p2, K in data:
            ts = []
            for _ in range(r):
                t0 = time.perf_counter()
                cv2.solvePnPRansac(X.reshape(-1, 1, 3), p2.reshape(-1, 1, 2), K, np.zeros((1, 4), np.float32), None, None, False, 100, 10.0, 0.99)
                ts.append(1e3 * (time.perf_counter() - t0))
            out.append(float(np.median(ts)))
        return out
    one = cv_ms(1, sets); allt = cv_ms(os.cpu_count() or 1, sets)
    syn_one = cv_ms(1, [syn], 1)[0]; syn_all = cv_ms(os.cpu_count() or 1, [syn], 1)[0]
    cv2.setNumThreads(-1)
    kernels = {"crazyhorse_%d" % k: pose_kernel_ms(lambda X=X, p2=p2, K=K: ctx.find_camera_pose(K, X, p2)) for k, (X, p2, K) in enumerate(sets)}
    if profile:
        kernels["synthetic_100000"] = pose_kernel_ms(lambda: ctx.find_camera_pose(syn[2], syn[0], syn[1]))
    name, pl = card()
    return {"metric": "pnp_ransac_pose_ms_per_call", "gpu_ms": gpu, "cv2_1thread_ms": one, "cv2_all_threads_ms": allt,
            "correspondences": [int(len(X)) for X, _, _ in sets], "gpu_median_ms": float(np.median(gpu)),
            "cv2_1thread_median_ms": float(np.median(one)), "cv2_all_threads_median_ms": float(np.median(allt)),
            "synthetic_100000_gpu_median_ms": float(np.median(t_syn)), "synthetic_100000_cv2_1thread_ms": syn_one,
            "synthetic_100000_cv2_all_threads_ms": syn_all, "kernel_ms_torch_profiler": kernels if profile else "not profiled",
            "card": name, "power_limit": pl, "cpu_threads": os.cpu_count()}


def measure_all(images=50, features=5000, points=1_000_000, reps=5, ctx=None, stages=("match", "triangulate", "essential"), profile=False):
    import torch
    from sfm_toy_library_b200 import capi
    own = ctx is None
    if own:
        torch.cuda.set_device(0); ctx = capi.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    flush = torch.empty(192 << 20, dtype=torch.uint8, device="cuda")
    out = []
    if "match" in stages:
        out += [measure_match(ctx, stream, flush, images, features, reps, "hamming"), measure_match(ctx, stream, flush, images, features, reps, "l2")]
    if "triangulate" in stages:
        out.append(measure_triangulate(ctx, stream, flush, points, reps))
    if "essential" in stages:
        out.append(measure_essential(ctx, profile=profile))
    if "homography" in stages:
        out.append(measure_homography(ctx, images))
    if "triangulate-pairs" in stages:
        out.append(measure_triangulate_pairs(ctx, profile=profile))
    if "pose" in stages:
        out.append(measure_pose(ctx, profile=profile))
    if own:
        ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=50)
    ap.add_argument("--features", type=int, default=5000)
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stages", default="match,triangulate,essential", help="comma-separated subset of match, triangulate, essential, homography, triangulate-pairs, pose")
    ap.add_argument("--no-profile", action="store_true", help="skip the torch.profiler kernel split of the essential, triangulate-pairs and pose stages")
    args = ap.parse_args()
    for line in measure_all(args.images, args.features, args.points, args.reps, stages=args.stages.split(","), profile=not args.no_profile):
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
