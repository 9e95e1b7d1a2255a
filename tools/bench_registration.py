"""Cost of a registration evaluation (usip_b200.evaluation.registration) on a synthetic KITTI test tree at real sizes
-- one JSON line.

  * per scan: the descriptor pass (ModelDescriptor.run_model at the detector's keypoints, batches of 8), from CUDA
    events over the whole test set;
  * usip_desc_match_f64 per 1000 pairs for the 8-value K sweep 4 .. 512 (KITTI's one-way 1-NN, and Oxford's k = 5
    union on the same descriptors);
  * usip_ransac_rt_f64 per 1000 pairs for the maxTrials sweep 50 .. 10000 on those matches.  The weights are random,
    so the matches are garbage and every (pair, K) runs to the cap: the worst case;
  * usip_ransac_rt_f64 per 1000 pairs on synthetic correspondences (512 per pair, 30 % inliers), where the adaptive
    stop ends most runs early;
  * end to end: pairs/s of Registration.run (host clock around a run that ends in a device synchronise).
The tree: --scans 20480-row scans (N = 16384, M = 512) in two sequences, each scan paired with its two successors.

    python tools/bench_registration.py [--scans 300] [--out profiles/registration_h100.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_pairgen import event_ms, gpu_info  # noqa: E402
from usip_b200 import ops  # noqa: E402
from usip_b200.evaluation import kitti_test_loader as ktl  # noqa: E402
from usip_b200.evaluation import registration as reg  # noqa: E402
from usip_b200.evaluation import repeatability as rep  # noqa: E402

KS = [4, 8, 16, 32, 64, 128, 256, 512]
TRIALS = list(reg.DEFAULT_MAX_TRIALS)


def synthetic_correspondences(P, n, ratio, seed):
    """P pairs of n correspondences of a random motion, a fraction `ratio` inliers (residual <= 0.3), the others
    3 .. 40 away -> kernel inputs with identity frames."""
    rng = np.random.RandomState(seed)
    xyz = np.zeros((2 * P, n, 3), np.float32)
    for p in range(P):
        t, q = ktl.random_rigid(rng)
        T = rep.gt_transform(t, q)
        x2 = rng.uniform(-40, 40, (n, 3))
        x1 = x2 @ T[:, :3].T + T[:, 3]
        dirs = rng.normal(size=(n, 3))
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        x1 += dirs * np.where(rng.rand(n) < ratio, rng.uniform(0, 0.3, n), rng.uniform(3, 40, n))[:, None]
        xyz[2 * p], xyz[2 * p + 1] = x1, x2
    matches = np.zeros((P, 1, n, 2), np.int32)
    matches[:, 0] = np.stack([np.arange(n), np.arange(n)], 1)
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return (c(xyz), c(np.full(2 * P, n, np.int32)), c(np.stack([np.arange(P) * 2, np.arange(P) * 2 + 1], 1)
                                                      .astype(np.int32)),
            c(np.broadcast_to(np.eye(3, 4), (P, 3, 3, 4))), c(matches), c(np.full((P, 1), n, np.int32)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=300)
    ap.add_argument("--rows", type=int, default=20480)
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--M", type=int, default=512)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from oracle import usip_oracle as orc
    from tests.util_gpu import load_params, make_opt
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    from usip_b200.models.keypoint_detector import ModelDetector
    info = gpu_info()
    opt = make_opt(batch_size=8, input_pc_num=a.N, node_num=a.M, ball_radius=2.0)
    det = ModelDetector(opt)
    load_params(det.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    det.freeze_model()
    torch.manual_seed(1)
    des = ModelDescriptor(opt)
    des.freeze_model()
    with tempfile.TemporaryDirectory() as root:
        counts = [a.scans // 2, a.scans - a.scans // 2]
        pairs = [[(i, j) for i in range(n) for j in (i + 1, i + 2) if j < n] for n in counts]
        txt, num, cal = (os.path.join(root, d) for d in ("txt", "numpy", "calib"))
        ktl.write_synthetic_kitti_test(txt, num, cal, counts, a.rows, pairs, seed=1)
        ev = reg.Registration(rep.KittiRepeatability(txt, num, cal, opt, seed=0, batch_size=8))
        S, P = len(ev.ev.source), len(ev.ev.pairs)
        ev.run(det, des, KS, max_trials=TRIALS)                 # warm-up: every shape, module loads
        torch.cuda.synchronize()

        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        desc_ms = 0.0
        for items, (pc, sn, node) in ev.ev.source.batches():
            k, _ = det.run_model(pc, sn, node)
            e0.record()
            des.run_model(pc, sn, k)
            e1.record()
            e1.synchronize()
            desc_ms += e0.elapsed_time(e1)
        L = min(ev.xyz.shape[1], KS[-1])
        xyz, desc = ev.xyz[:, :L].contiguous(), ev.desc[:, :L].contiguous()
        count = torch.clamp(ev.count, max=L).to(torch.int32).contiguous()
        pairs_d = torch.from_numpy(ev.ev.pairs).cuda()
        frames_d = torch.from_numpy(ev.ev.frames).cuda()
        match1 = event_ms(lambda: ops.desc_match(desc, count, pairs_d, KS, 1), 5)
        match5 = event_ms(lambda: ops.desc_match(desc, count, pairs_d, KS, 5), 5)
        m, n = ops.desc_match(desc, count, pairs_d, KS, 1)
        ransac = event_ms(lambda: ops.ransac_rt(xyz, count, pairs_d, frames_d, m, n, TRIALS), 3)
        capped = ops.ransac_rt(xyz, count, pairs_d, frames_d, m, n, TRIALS)["trialcount"][:, :, -1]
        syn = synthetic_correspondences(1000, 512, 0.3, 2)
        ransac30 = event_ms(lambda: ops.ransac_rt(*syn, TRIALS), 3)
        syn_tc = ops.ransac_rt(*syn, TRIALS)["trialcount"][:, 0, -1].float().mean().item()
        t0 = time.perf_counter()
        res = ev.run(det, des, KS, max_trials=TRIALS)
        torch.cuda.synchronize()
        e2e = time.perf_counter() - t0
    line = {
        "what": "registration evaluation, synthetic KITTI test tree",
        "gpu": info, "scans": S, "pairs": P, "scan_rows": a.rows, "N": a.N, "M": a.M, "keypoint_nums": KS,
        "max_trials": TRIALS,
        "descriptor_per_scan_ms": desc_ms / S,
        "match_ms_per_1000_pairs": {"k1_kitti": match1 / P * 1000, "k5_union_oxford": match5 / P * 1000},
        "ransac_ms_per_1000_pairs": {
            "random_weights_kitti_matches": ransac / P * 1000,
            "random_weights_share_of_runs_at_cap": float((capped == TRIALS[-1] + 1).float().mean().item()),
            "synthetic_512_matches_30pct_inliers": ransac30,
            "synthetic_mean_trialcount_at_10000": syn_tc},
        "end_to_end_pairs_per_s": P / e2e,
        "recall_at_K512_T10000": float(res.recall[-1, -1]),
        "reference": "evaluate_kitti.m's parfor needs MATLAB: not measured",
    }
    print(json.dumps(line))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
