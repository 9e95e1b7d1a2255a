"""Cost of a repeatability evaluation (usip_b200.evaluation.repeatability) on a synthetic KITTI test tree at real sizes
-- one JSON line.

  * per scan: the device-mode test-cloud build (file load, upload, subsample, FPS, gather), the detector pass
    (ModelDetector.run_model, batches of 8 as save_keypoints.py) and the selection (one stable sort or NMS over all
    scans), each from CUDA events over the whole test set;
  * scoring: usip_repeatability_f64 per 1000 pairs for the 8-value K sweep 4 .. 512;
  * end to end: scans/s of KittiRepeatability.run (host clock around a run that ends in a device synchronise).
The tree: --scans 20480-row scans (N = 16384, M = 512) in two sequences, each scan paired with its two successors.
The detector is randomly initialised: its keypoints have no meaning, only the cost matters.

    python tools/bench_repeatability.py [--scans 300] [--out profiles/repeatability_h100.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_pairgen import event_ms, gpu_info  # noqa: E402
from usip_b200 import ops  # noqa: E402
from usip_b200.evaluation import kitti_test_loader as ktl  # noqa: E402
from usip_b200.evaluation import repeatability as rep  # noqa: E402

KS = [4, 8, 16, 32, 64, 128, 256, 512]


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
    from usip_b200.models.keypoint_detector import ModelDetector
    info = gpu_info()
    opt = make_opt(batch_size=8, input_pc_num=a.N, node_num=a.M)
    md = ModelDetector(opt)
    load_params(md.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    md.freeze_model()
    with tempfile.TemporaryDirectory() as root:
        counts = [a.scans // 2, a.scans - a.scans // 2]
        pairs = [[(i, j) for i in range(n) for j in (i + 1, i + 2) if j < n] for n in counts]
        txt, num, cal = (os.path.join(root, d) for d in ("txt", "numpy", "calib"))
        ktl.write_synthetic_kitti_test(txt, num, cal, counts, a.rows, pairs, seed=1)
        ev = rep.KittiRepeatability(txt, num, cal, opt, seed=0, batch_size=8)
        S, P = len(ev.source), len(ev.pairs)
        ev.run(md, KS)                                        # warm-up: every shape, module loads, graph captures
        torch.cuda.synchronize()

        ev_b = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        detect_ms = 0.0
        kp = torch.empty((S, 3, a.M), device="cuda"); sg = torch.empty((S, a.M), device="cuda")
        for items, (pc, sn, node) in ev.source.batches():
            ev_b[1].record()
            k, s = md.run_model(pc, sn, node)
            ev_b[2].record()
            kp[items[0]:items[-1] + 1] = k; sg[items[0]:items[-1] + 1] = s
            ev_b[2].synchronize()
            detect_ms += ev_b[1].elapsed_time(ev_b[2])
        t0 = time.perf_counter()
        for items in [list(range(i, min(i + 8, S))) for i in range(0, S, 8)]:
            ev.source.build(items)
        torch.cuda.synchronize()
        build_ms = (time.perf_counter() - t0) * 1e3
        sel0 = event_ms(lambda: rep.select_order(kp, sg, 0.0), 20)
        sel1 = event_ms(lambda: rep.select_order(kp, sg, 1.0), 20)
        order, count = rep.select_order(kp, sg, 0.0)
        pairs_d = torch.from_numpy(ev.pairs).cuda(); frames_d = torch.from_numpy(ev.frames).cuda()
        score = event_ms(lambda: ops.repeatability(kp, order, count, pairs_d, frames_d, KS, 0.5), 20)
        t0 = time.perf_counter()
        res = ev.run(md, KS)
        torch.cuda.synchronize()
        e2e = time.perf_counter() - t0
    line = {
        "what": "repeatability evaluation, synthetic KITTI test tree",
        "gpu": info, "scans": S, "pairs": P, "scan_rows": a.rows, "N": a.N, "M": a.M, "keypoint_nums": KS,
        "per_scan_ms": {"cloud_build_host_clock": build_ms / S, "detect": detect_ms / S,
                        "select_sort": sel0 / S, "select_nms_r1": sel1 / S},
        "score_ms_per_1000_pairs": score / P * 1000,
        "end_to_end_scans_per_s": S / e2e,
        "mean_repeatability": [round(float(x), 4) for x in res.mean_repeatability],
        "reference_loader": "KittiTestLoader.__getitem__ host time: not measured here (the reference tree is not on the "
                            "GPU host); eval_rep.m needs MATLAB: not measured",
    }
    print(json.dumps(line))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
