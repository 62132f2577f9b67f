"""Device time of sfmb200_triangulate_device on 1 M points at fixture world scale x1, x10 and x100, i.e. with every point on the
closed-form null vector, a mix, and every point on the Jacobi fallback (csrc/dlt_math.cuh).  CUDA events around the call after a
warm-up; the card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/bench_triangulate_paths.py [--points 1000000] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch

    import dlt_util as du
    from sfm_toy_library_b200 import capi
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    ctx = capi.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)           # the events go on the context's own stream
    m = args.points
    out = {"metric": "triangulate_device_ms_per_call", "points": m}
    for s in (1, 10, 100):
        sc = du.fixture_scaled(s, m, seed=0)
        A = du.triangulation_matrices(sc["K"], sc["Pl"], sc["Pr"], sc["ptsL"][:20000], sc["ptsR"][:20000])
        _, ok, _ = du.host_null_vectors(A)
        dl = torch.from_numpy(sc["ptsL"]).cuda(); dr = torch.from_numpy(sc["ptsR"]).cuda()
        dX = torch.empty(3 * m, dtype=torch.float32, device="cuda"); dk = torch.empty(m, dtype=torch.uint8, device="cuda")
        dn = torch.empty(1, dtype=torch.int32, device="cuda")
        call = lambda: ctx.triangulate_device(sc["K"], sc["Pl"], sc["Pr"], dl.data_ptr(), dr.data_ptr(), None, None, m, dX.data_ptr(),
                                              dk.data_ptr(), dn.data_ptr())
        for _ in range(3):
            call()
        ctx.synchronize(); torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            ctx.synchronize(); e0.record(stream); call(); e1.record(stream); ctx.synchronize(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        out[f"x{s}"] = {"median_ms": float(np.median(ts)), "min_ms": float(np.min(ts)), "max_ms": float(np.max(ts)),
                        "host_model_declined_share": float((~ok).mean())}
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    out.update(card=torch.cuda.get_device_name(0), power_limit=pl)
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
