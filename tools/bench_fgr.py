"""Fast Global Registration timings on one GPU, against RANSAC in the same job.

Workload: the Redwood-shaped synthetic tree of tools/bench_registration_indoor.py (the four scenes, 5,280 pairs over all
i < j, 30,000-row fragments, 512 keypoints with 128-D random descriptors each) and the default K sweep 4 .. 512.
Reports, each from CUDA events around the launches:
  mutual_match_ms_per_1000_pairs and fgr_ms_per_1000_pairs (the whole K sweep, first 1000 pairs), with the status mix;
  match_ms_per_1000_pairs and ransac_ms_per_1000_pairs at maxTrials 1000 and 30000 (k = 5 matches, same pairs and Ks);
  end-to-end IndoorRegistration.score(solver="fgr") over all 5,280 pairs (host clock, ends in a copy);
  synthetic correspondences with a known inlier fraction (512 matches per pair, K = 512): 1.0 saturates the 10,000-tuple
  cap, the worst case; 0.5 and 0.25 are typical; random descriptors above are the cheap case (few tuples, no iterations).
The card's name and power limit are read in the same run.  `python tools/bench_fgr.py --out FILE`."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_registration_indoor import card, timed  # noqa: E402
from usip_b200 import ops  # noqa: E402
from usip_b200.evaluation import indoor_registration as idr  # noqa: E402
from usip_b200.evaluation import indoor_test_loader as itl  # noqa: E402
from usip_b200.evaluation import registration as reg  # noqa: E402
from usip_b200.evaluation.kitti_test_loader import random_rigid  # noqa: E402
from usip_b200.evaluation.repeatability import DEFAULT_KEYPOINT_NUMS, gt_transform  # noqa: E402


def _status_mix(status):
    s = status.cpu().numpy().ravel()
    return {str(v): int((s == v).sum()) for v in range(5) if (s == v).any()}


def synthetic(P, n, inlier_fraction, rng, dev):
    """P pairs of n correspondences (i, i): fragment 2 a rigid copy of fragment 1, then the first (1 - f) n matches
    re-pointed at random rows -> the arguments of ops.fgr."""
    a = rng.uniform(-3, 3, (P, n, 3))
    xyz = np.empty((2 * P, n, 3), np.float32)
    for p in range(P):
        T = gt_transform(*random_rigid(rng))
        xyz[2 * p] = a[p]
        xyz[2 * p + 1] = (a[p] - T[:, 3]) @ T[:, :3]
    m = np.stack([np.arange(n), np.arange(n)], 1)[None, None].repeat(P, 0).copy()
    k = int(round((1 - inlier_fraction) * n))
    m[:, 0, :k, 1] = rng.randint(0, n, (P, k))
    count = np.full(2 * P, n, np.int32)
    pairs = np.arange(2 * P, dtype=np.int32).reshape(P, 2)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    return t(xyz), t(count), t(pairs), t(m.astype(np.int32)), t(np.full((P, 1), n, np.int32))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/fgr_h100.json")
    ap.add_argument("--rows", type=int, default=30000)
    ap.add_argument("--keypoints", type=int, default=512)
    ap.add_argument("--synthetic-pairs", type=int, default=1000)
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = card()
    tmp = tempfile.mkdtemp(prefix="usip_fgr_")
    npy, gt, tree = (os.path.join(tmp, x) for x in ("npy", "gt", "tree"))
    pairs = {s: [(i, i + 2) for i in range(0, n - 2, 5)] for s, n in itl.REDWOOD_SCENES}
    itl.write_synthetic_redwood(npy, gt, a.rows, pairs, seed=0)
    rng = np.random.RandomState(0)
    L, D = a.keypoints, 128
    for s, n in itl.REDWOOD_SCENES:
        os.makedirs(os.path.join(tree, s), exist_ok=True)
        for f in range(n):
            x = np.load(os.path.join(npy, s, "%d.npy" % f))[:L, :3]
            np.concatenate([x, rng.normal(size=(L, D))], 1).astype(np.float32).tofile(os.path.join(tree, s, "%d.bin" % f))
    ev = idr.IndoorRegistration.redwood(npy, gt, reg.descriptor_opt("redwood"))
    ev.read_descriptor_tree(tree, D)
    ks = [k for k in DEFAULT_KEYPOINT_NUMS if k <= L]
    ts = list(idr.DEFAULT_MAX_TRIALS)

    # components on the first 1000 pairs of livingroom1 + livingroom2, the whole K sweep
    fp = [(s, p) for s in ev.scenes[:2] for p in ev.scene_pairs(s)][:1000]
    dev = ev.xyz.device
    pr = torch.tensor([[ev.index[(s, int(i))], ev.index[(s, int(j))]] for s, (i, j) in fp], dtype=torch.int32,
                      device=dev)
    frames = torch.from_numpy(np.broadcast_to(np.eye(3, 4), (len(fp), 3, 3, 4)).copy()).to(dev)
    xyz, desc, count = ev.xyz.contiguous(), ev.desc.contiguous(), ev.count
    per = 1000.0 / len(fp)
    t_mut, (mm, mn) = timed(lambda: ops.desc_match_mutual(desc, count, pr, ks))
    t_fgr, fo = timed(lambda: ops.fgr(xyz, count, pr, ks, mm, mn, idr.INLIER_THRESHOLD, 0))
    t_match, (m, n) = timed(lambda: ops.desc_match(desc, count, pr, ks, idr.MATCH_K))
    t_ransac, _ = timed(lambda: ops.ransac_rt(xyz, count, pr, frames, m, n, ts, idr.INLIER_THRESHOLD, 0), reps=1)
    real = {"mutual_match_ms_per_1000_pairs": t_mut * per, "fgr_ms_per_1000_pairs": t_fgr * per,
            "fgr_status_counts": _status_mix(fo["status"]), "fgr_max_tuples": int(fo["n_tuples"].max().item()),
            "match_k5_ms_per_1000_pairs": t_match * per, "ransac_1000_and_30000_ms_per_1000_pairs": t_ransac * per}

    # end to end over every pair
    ev.score(ks, pairs="gt", solver="fgr")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = ev.score(ks, pairs="all", solver="fgr")
    t_e2e = time.perf_counter() - t0
    n_pairs = sum(len(r["pairs"]) for r in res.per_scene.values())

    # synthetic correspondences with a known inlier fraction, K = n = 512
    syn = {}
    for f in (1.0, 0.5, 0.25):
        args = synthetic(a.synthetic_pairs, L, f, rng, dev)
        t_s, so = timed(lambda: ops.fgr(args[0], args[1], args[2], [L], args[3], args[4], idr.INLIER_THRESHOLD, 0),
                        reps=1)
        syn["inlier_fraction_%g" % f] = {
            "fgr_ms_per_1000_pairs": t_s * 1000.0 / a.synthetic_pairs, "status_counts": _status_mix(so["status"]),
            "mean_tuples": float(so["n_tuples"].double().mean().item()),
            "mean_inliers": float(so["n_inliers"].double().mean().item())}
    rec = {
        "gpu": name, "power_limit": power,
        "workload": {"scenes": len(itl.REDWOOD_SCENES), "pairs": n_pairs, "fragment_rows": a.rows, "keypoints": L,
                     "descriptor_dim": D, "keypoint_nums": ks, "ransac_max_trials": ts,
                     "synthetic_pairs": a.synthetic_pairs, "synthetic_matches": L},
        "random_descriptors_first_1000_pairs": real,
        "end_to_end_fgr_s": t_e2e, "end_to_end_fgr_pairs_per_s": n_pairs / t_e2e,
        "synthetic_correspondences": syn,
        "note": "random descriptors give few tuples, so most (pair, K) entries stop before the iterations; the "
                "synthetic inlier fraction 1.0 saturates the 10,000-tuple cap and runs all 640 iterations everywhere",
    }
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
