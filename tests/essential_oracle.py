"""TEST INFRASTRUCTURE ONLY: CPU restatement of the selection half of OpenCV's RANSAC (RANSACPointSetRegistrator::run and
RANSACUpdateNumIters, OpenCV calib3d ptsetreg.cpp), fed with per-solution inlier counts already scored in sample order.  The
device replays the same loop in essential_select_kernel (csrc/essential.cu); tests/test_gpu_essential.py compares the two on
the traces of real calls, tests/test_five_point_host.py pins this restatement on hand-computed cases."""
import math
import sys

import numpy as np


def ransac_update_num_iters(p, ep, model_points, max_iters):
    """RANSACUpdateNumIters: samples needed for confidence p at outlier ratio ep, capped at max_iters (the current budget)."""
    p = min(max(p, 0.0), 1.0)
    ep = min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, sys.float_info.min)
    denom = 1.0 - math.pow(1.0 - ep, model_points)
    if denom < sys.float_info.min:
        return 0
    num = math.log(num)
    denom = math.log(denom)
    return max_iters if denom >= 0 or -num >= max_iters * (-denom) else int(round(num / denom))      # cvRound: half to even


def sequential_select(nsol, counts, n, max_iters=1000, confidence=0.999, model_points=5):
    """RANSACPointSetRegistrator::run's loop over solutions already scored, in sample order: nsol [S] solutions per sample,
    counts [sum nsol] inliers per solution.  A solution replaces the best only if its count exceeds max(best, model_points - 1);
    each improvement recomputes the sample budget.  Returns (index of the best solution in counts or -1, its count, samples visited)."""
    niters = max(max_iters, 1); best = -1; max_good = 0; off = np.concatenate([[0], np.cumsum(nsol)]).astype(int)
    it = 0
    while it < niters and it < len(nsol):
        for k in range(int(nsol[it])):
            g = int(counts[off[it] + k])
            if g > max(max_good, model_points - 1):
                best = int(off[it] + k); max_good = g
                niters = ransac_update_num_iters(confidence, (n - g) / n, model_points, niters)
        it += 1
    return best, max_good, it
