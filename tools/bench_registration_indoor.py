"""Indoor registration timings: a Redwood-shaped synthetic tree (the four scenes, 57 + 47 + 53 + 50 fragments, 5,280
pairs over all i < j, 30,000-row fragments, 512 keypoints with 128-D descriptors each) and a 3DMatch-shaped scene of
250,000-row fragments.  Reports, each from CUDA events around the launches on one GPU:
  match_ms_per_1000_pairs, ransac_ms_per_1000_pairs (maxTrials 1000 and 30000 in one stream), info_ms_per_1000_pairs,
  overlap_ms_per_1000_jobs (Redwood-sized and 3DMatch-sized fragments), the jobs that passed the inlier-ratio filter in
  the end-to-end run, and end-to-end pairs/s of IndoorRegistration.score(pairs="all") (host clock, ends in a copy).
The card's name and power limit are read in the same run.  `python tools/bench_registration_indoor.py --out FILE`."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from usip_b200 import ops  # noqa: E402
from usip_b200.evaluation import indoor_registration as idr  # noqa: E402
from usip_b200.evaluation import indoor_test_loader as itl  # noqa: E402
from usip_b200.evaluation import registration as reg  # noqa: E402
from usip_b200.evaluation.kitti_test_loader import random_rigid  # noqa: E402
from usip_b200.evaluation.repeatability import gt_transform  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True).strip().splitlines()[0]
        name, power = [v.strip() for v in out.split(",")]
        return name, power
    except Exception as e:                                      # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/registration_indoor_h100.json")
    ap.add_argument("--rows", type=int, default=30000)
    ap.add_argument("--rows-3dmatch", type=int, default=250000)
    ap.add_argument("--keypoints", type=int, default=512)
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = card()
    tmp = tempfile.mkdtemp(prefix="usip_reg_indoor_")
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
    opt = reg.descriptor_opt("redwood")
    ev = idr.IndoorRegistration.redwood(npy, gt, opt)
    ev.read_descriptor_tree(tree, D)
    ks, ts = [L], list(idr.DEFAULT_MAX_TRIALS)

    # components, on the first 1000 pairs of livingroom1 + livingroom2
    fp = [(s, p) for s in ev.scenes[:2] for p in ev.scene_pairs(s)][:1000]
    dev = ev.xyz.device
    pr = torch.tensor([[ev.index[(s, int(i))], ev.index[(s, int(j))]] for s, (i, j) in fp], dtype=torch.int32,
                      device=dev)
    frames = torch.from_numpy(np.broadcast_to(np.eye(3, 4), (len(fp), 3, 3, 4)).copy()).to(dev)
    xyz, desc, count = ev.xyz.contiguous(), ev.desc.contiguous(), ev.count
    t_match, (m, n) = timed(lambda: ops.desc_match(desc, count, pr, ks, idr.MATCH_K))
    t_ransac, out = timed(lambda: ops.ransac_rt(xyz, count, pr, frames, m, n, ts, idr.INLIER_THRESHOLD, 0))
    t_info, _ = timed(lambda: ops.ransac_info(xyz, count, pr, frames, m, n, ts, out["best_trial"], out["status"],
                                              idr.INLIER_THRESHOLD, 0))
    # overlap: 1000 jobs over livingroom1's fragments, random rigid maps near the identity
    frag, offsets, where = ev._fragments(ev.scenes[0])
    nf = len(offsets) - 1
    jobs = np.array([(j % nf, (j * 7 + 1) % nf) for j in range(1000)], np.int32)
    maps = np.array([gt_transform(*random_rigid(rng)) for _ in range(1000)])
    maps[:, :, 3] *= 0.05
    maps_d = torch.from_numpy(maps).to(dev)
    t_ov, _ = timed(lambda: ops.fragment_overlap(frag, offsets, jobs, maps_d))
    # a 3DMatch-shaped scene: 20 fragments of 250,000 rows, all 190 pairs
    big = [itl.synthetic_fragment(100 + f, a.rows_3dmatch)[:, :3] for f in range(20)]
    big_off = np.concatenate([[0], np.cumsum([len(b) for b in big])]).astype(np.int64)
    big_d = torch.from_numpy(np.concatenate(big)).to(dev)
    bj = np.array([(i, j) for i in range(20) for j in range(i + 1, 20)], np.int32)
    bm = torch.from_numpy(np.array([gt_transform(*random_rigid(rng)) * [1, 1, 1, 0.05] for _ in bj])).to(dev)
    t_ov_big, _ = timed(lambda: ops.fragment_overlap(big_d, big_off, bj, bm), reps=1)

    # end to end: every pair of the four scenes
    ev.score(ks, ts, pairs="gt")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = ev.score(ks, ts, pairs="all")
    t_e2e = time.perf_counter() - t0
    n_pairs = sum(len(r["pairs"]) for r in res.per_scene.values())
    n_jobs = int(sum((r["inlier_ratio"] > idr.INLIER_RATIO_THRESHOLD).sum() for r in res.per_scene.values()))
    rec = {
        "gpu": name, "power_limit": power,
        "workload": {"scenes": len(itl.REDWOOD_SCENES), "pairs": n_pairs, "fragment_rows": a.rows, "keypoints": L,
                     "descriptor_dim": D, "max_trials": ts, "match_k": idr.MATCH_K,
                     "overlap_3dmatch": {"fragments": 20, "rows": a.rows_3dmatch, "jobs": len(bj)}},
        "match_ms_per_1000_pairs": t_match * 1000 / len(fp),
        "ransac_ms_per_1000_pairs": t_ransac * 1000 / len(fp),
        "info_ms_per_1000_pairs": t_info * 1000 / len(fp),
        "overlap_ms_per_1000_jobs_30k_rows": t_ov,
        "overlap_ms_per_1000_jobs_250k_rows": t_ov_big * 1000 / len(bj),
        "end_to_end_s": t_e2e, "end_to_end_pairs_per_s": n_pairs / t_e2e,
        "jobs_past_inlier_ratio_filter": n_jobs,
        "note": "synthetic fragments are independent random rooms, so few jobs pass the inlier-ratio filter end to end; "
                "the overlap rows time forced jobs",
    }
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
