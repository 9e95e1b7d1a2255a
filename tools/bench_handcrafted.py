"""Time the handcrafted keypoint baselines (csrc/handcrafted.cu) per scan: the grid build, the saliency or response
pass, the non-maximum pass and the selection, with the mean neighbourhood size the passes walk, for ISS at the KITTI
shape and radii and for Harris-3D at the KITTI and Redwood shapes; then KittiRepeatability.run(IssDetector())
end to end on a synthetic KITTI test tree.  The clouds are synthetic (synthetic_scan: 80 m x 80 m, height sigma 1.5 m;
synthetic_fragment: a 4 m cube), not KITTI's or Redwood's density, and the times scale with |N_r|.

    python tools/bench_handcrafted.py [--out profiles/handcrafted_h100.json]
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
from usip_b200.data.kitti_detector_loader import synthetic_scan  # noqa: E402
from usip_b200.evaluation import kitti_test_loader as ktl  # noqa: E402
from usip_b200.evaluation import repeatability as rep  # noqa: E402
from usip_b200.evaluation.handcrafted import IssDetector  # noqa: E402
from usip_b200.evaluation.indoor_test_loader import synthetic_fragment  # noqa: E402

KS = [4, 8, 16, 32, 64, 128, 256, 512]
REPS = 20


def _clouds(make, B, N):
    return torch.from_numpy(np.stack([make(s, N)[:, :3].T for s in range(B)]).astype(np.float32)).cuda().contiguous()


def _phases(pc, method, radii, M):
    B = pc.shape[0]
    grid = ops.hc_grid(pc)
    t = {"grid": event_ms(lambda: ops.hc_grid(pc), REPS)}
    if method == "iss":
        rs, rn = radii
        sal, cnt, _ = ops.iss_saliency(grid, rs, 0.975, 0.975, 5)
        t["saliency"] = event_ms(lambda: ops.iss_saliency(grid, rs, 0.975, 0.975, 5), REPS)
        flag, cnt_n = ops.hc_nonmax(grid, sal, rn, 0.0, True, 5)
        t["non_max"] = event_ms(lambda: ops.hc_nonmax(grid, sal, rn, 0.0, True, 5), REPS)
    else:
        (r,) = radii
        resp, cnt, _ = ops.harris3d_response(grid, r)
        t["normals_and_response"] = event_ms(lambda: ops.harris3d_response(grid, r), REPS)
        flag, cnt_n = ops.hc_nonmax(grid, resp, r, 0.001, False, 1)
        t["non_max"] = event_ms(lambda: ops.hc_nonmax(grid, resp, r, 0.001, False, 1), REPS)
    _, det = ops.hc_select(flag, B, pc.shape[2], M, 0, 0)
    t["selection"] = event_ms(lambda: ops.hc_select(flag, B, pc.shape[2], M, 0, 0), REPS)
    torch.cuda.synchronize()
    return {"per_scan_ms": {k: v / B for k, v in t.items()},
            "total_per_scan_ms": sum(t.values()) / B,
            "mean_neighbours_per_query": float(cnt.double().mean()),
            "mean_neighbours_per_query_non_max": float(cnt_n.double().mean()),
            "mean_detected_per_scan": float(det.double().mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=96)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    B, M = 8, 512
    kitti = _clouds(synthetic_scan, B, 16384)
    redwood = _clouds(synthetic_fragment, B, 10240)
    out = {
        "what": "handcrafted keypoint baselines, per scan, B = 8 clouds per call",
        "gpu": info,
        "iss_kitti": dict(_phases(kitti, "iss", (2.0, 2.0), M), N=16384, salient_radius=2.0, non_max_radius=2.0),
        "harris_kitti": dict(_phases(kitti, "harris", (1.0,), M), N=16384, radius=1.0),
        "harris_redwood": dict(_phases(redwood, "harris", (0.3,), M), N=10240, radius=0.3,
                               radius_note="assumed: the reference states no Harris radius for Redwood"),
        "clouds": "synthetic_scan (80 m x 80 m, height sigma 1.5 m) and synthetic_fragment (4 m cube): not the density "
                  "of real KITTI or Redwood scans; the pass times scale with the neighbours per query",
        "pcl_reference": "not measured: PCL and the reference's PCLKeypoint module are not available, no estimate given",
    }
    from tests.util_gpu import make_opt
    opt = make_opt(batch_size=8, input_pc_num=16384, node_num=M)
    with tempfile.TemporaryDirectory() as root:
        counts = [a.scans // 2, a.scans - a.scans // 2]
        pairs = [[(i, j) for i in range(n) for j in (i + 1, i + 2) if j < n] for n in counts]
        txt, num, cal = (os.path.join(root, d) for d in ("txt", "numpy", "calib"))
        ktl.write_synthetic_kitti_test(txt, num, cal, counts, 20480, pairs, seed=1)
        ev = rep.KittiRepeatability(txt, num, cal, opt, seed=0, batch_size=8)
        det = IssDetector()
        ev.run(det, KS)                                       # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ev.run(det, KS)
        torch.cuda.synchronize()
        e2e = time.perf_counter() - t0
        out["kitti_repeatability_iss_end_to_end"] = {
            "scans": len(ev.source), "pairs": len(ev.pairs), "scans_per_s": len(ev.source) / e2e,
            "detected": det.count_summary(),
            "mean_repeatability": [round(float(x), 4) for x in res.mean_repeatability]}
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
