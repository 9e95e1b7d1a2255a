"""Cost of repeatability evaluation on the rotated ModelNet40, Redwood and 3DMatch test sets, and of usip_cloud_subsample
at every scan length -- one JSON line.

  * per dataset, on a synthetic tree at the reference's shapes (ModelNet: 10000-point objects, N = 5000, S = 3; Redwood
    and 3DMatch: N = 10240, S = 4, fragments of --redwood-rows / --match3d-rows rows, the latter above the one-CTA
    subsample limit): the per-scan device-mode cloud build (host clock around whole batches ending in a synchronise),
    the detector pass (CUDA events) and the scoring launch for the K sweep 4 .. 512 (CUDA events);
  * usip_cloud_subsample for 8 clouds (N = 10240, N/2 candidates) at 20480 rows (one-CTA kernel) and at 60000, 250000
    and 1000000 rows (cluster kernel), called through the C ABI with preallocated outputs, CUDA events over --launches
    back-to-back calls;
  * with --parent-lib (a libusip_b200.so of an earlier build), the same 20480-row call through that library, timed in
    alternating rounds with this build's, so the one-CTA path can be compared in one job.
The detector is randomly initialised: its keypoints have no meaning, only the cost matters.

    python tools/bench_repeatability_indoor.py [--out profiles/repeatability_indoor_h100.json] [--parent-lib PATH]
"""
import argparse
import ctypes
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
from usip_b200.evaluation import indoor_test_loader as itl  # noqa: E402
from usip_b200.evaluation import modelnet_test_loader as mtl  # noqa: E402
from usip_b200.evaluation import repeatability as rep  # noqa: E402

KS = [4, 8, 16, 32, 64, 128, 256, 512]


def _evaluator(name, root, a):
    opt = rep.detector_opt(name)
    if name == "modelnet":
        names = ["obj_%04d" % i for i in range(a.modelnet_objects)]
        os.makedirs(os.path.join(root, "normal"))
        mtl.write_synthetic_modelnet40_normal(os.path.join(root, "normal"), names, 10000, seed=1)
        mtl.write_rotated_modelnet(os.path.join(root, "normal"), os.path.join(root, "tree"), seed=1)
        return rep.ModelNetRepeatability(os.path.join(root, "tree"), opt, batch_size=4), opt
    if name == "redwood":
        scenes = [("livingroom1", a.fragments // 2), ("office1", a.fragments - a.fragments // 2)]
        pairs = {s: [(i, i + 1) for i in range(n - 1)] for s, n in scenes}
        itl.write_synthetic_redwood(os.path.join(root, "npy"), os.path.join(root, "gt"), a.redwood_rows, pairs,
                                    seed=1, scenes=scenes)
        return rep.RedwoodRepeatability(os.path.join(root, "npy"), os.path.join(root, "gt"), opt, batch_size=8,
                                        scenes=scenes), opt
    scenes = itl.MATCH3D_SCENES[:2]
    frames = {s: tuple(range(n)) for s, n in zip(scenes, (a.fragments // 2, a.fragments - a.fragments // 2))}
    pairs = {s: [(i, i + 1) for i in range(len(f) - 1)] for s, f in frames.items()}
    itl.write_synthetic_3dmatch(root, frames, a.match3d_rows, pairs, seed=1)
    return rep.Match3DRepeatability(root, opt, batch_size=8, scenes=scenes), opt


def bench_dataset(name, a):
    from oracle import usip_oracle as orc
    from tests.util_gpu import load_params
    from usip_b200.models.keypoint_detector import ModelDetector
    with tempfile.TemporaryDirectory() as root:
        ev, opt = _evaluator(name, root, a)
        md = ModelDetector(opt)
        load_params(md.detector, orc.init_detector_params(S=int(opt.surface_normal_len), seed=1, randomize_bn=True))
        md.freeze_model()
        S, P = len(ev.source), len(ev.pairs)
        ev.run(md, KS)                                        # warm-up: every shape, module loads
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _items, out in ev.source.batches():
            pass
        torch.cuda.synchronize()
        build_ms = (time.perf_counter() - t0) * 1e3
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        detect_ms = 0.0
        for _items, (pc, sn, node) in ev.source.batches():
            e0.record()
            md.run_model(pc, sn, node)
            e1.record()
            e1.synchronize()
            detect_ms += e0.elapsed_time(e1)
        ev.detect(md)
        pairs_d = torch.from_numpy(ev.pairs).cuda(); frames_d = torch.from_numpy(ev.frames).cuda()
        score = event_ms(lambda: ops.repeatability(ev.keypoints, ev.order, ev.count, pairs_d, frames_d, KS, 0.5), 20)
        rows = max(len(x) for x in ev.source.load(list(range(min(S, 8)))))
    return {"scans": S, "pairs": P, "N": int(opt.input_pc_num), "S": int(opt.surface_normal_len),
            "batch_size": ev.source.batch_size, "scan_rows": rows,
            "per_scan_ms": {"cloud_build_host_clock": build_ms / S, "detect": detect_ms / S},
            "score_ms": score}


def _subsample_case(rows, clouds=8, N=10240):
    scans = torch.from_numpy(np.random.RandomState(rows).uniform(-2, 2, (rows * clouds // 2, 4)).astype(np.float32))
    offsets = torch.arange(0, rows * clouds // 2 + 1, rows, dtype=torch.int64)
    soc = torch.from_numpy(np.repeat(np.arange(clouds // 2, dtype=np.int32), 2))
    return scans.cuda(), offsets.cuda(), soc.cuda(), N


def _call(lib, scans, offsets, soc, rows, N, outs):
    """usip_cloud_subsample through a library handle with preallocated outputs: the same host cost for every build."""
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = lib.usip_cloud_subsample(p(scans), scans.shape[1], p(offsets), p(soc), rows, soc.shape[0] // 2, N, N // 2, 0,
                                  ctypes.c_double(0.0), ctypes.c_uint64(0), ctypes.c_uint64(0), *[p(o) for o in outs],
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc


def _outs(clouds, N):
    return [torch.empty((clouds, N), dtype=torch.int32, device="cuda"),
            torch.empty((clouds, N // 2), dtype=torch.int32, device="cuda"),
            torch.empty((clouds,), dtype=torch.int32, device="cuda"), torch.empty((clouds,), dtype=torch.int32, device="cuda")]


def bench_subsample(a):
    from usip_b200 import _lib
    this = _lib.load()
    out = {}
    for rows in (20480, 60000, 250000, 1000000):
        scans, offsets, soc, N = _subsample_case(rows)
        outs = _outs(8, N)
        f = lambda: _call(this, scans, offsets, soc, rows, N, outs)
        f()
        out[str(rows)] = {"kernel": "one-CTA" if rows <= ops.pair_max_scan_rows() else "cluster",
                          "ms_per_call": event_ms(f, a.launches)}
    if a.parent_lib:
        parent_lib = ctypes.CDLL(a.parent_lib)
        scans, offsets, soc, N = _subsample_case(20480)
        mine_out, parent_out = _outs(8, N), _outs(8, N)
        mine = lambda: _call(this, scans, offsets, soc, 20480, N, mine_out)
        parent = lambda: _call(parent_lib, scans, offsets, soc, 20480, N, parent_out)
        parent(); mine()
        torch.cuda.synchronize()
        same = all(torch.equal(x, y) for x, y in zip(mine_out, parent_out))
        rounds = {"this": [], "parent": []}
        for _ in range(a.rounds):
            rounds["parent"].append(event_ms(parent, a.launches))
            rounds["this"].append(event_ms(mine, a.launches))
        out["20480_vs_parent"] = {"outputs_bit_identical": bool(same),
                                  "this_ms_median": float(np.median(rounds["this"])),
                                  "parent_ms_median": float(np.median(rounds["parent"])),
                                  "this_ms_rounds": rounds["this"], "parent_ms_rounds": rounds["parent"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modelnet-objects", type=int, default=64)
    ap.add_argument("--fragments", type=int, default=32)
    ap.add_argument("--redwood-rows", type=int, default=30000)
    ap.add_argument("--match3d-rows", type=int, default=250000)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    line = {"what": "repeatability evaluation on rotated ModelNet40 / Redwood / 3DMatch synthetic trees, and "
                    "usip_cloud_subsample by scan length",
            "gpu": gpu_info(), "keypoint_nums": KS,
            "datasets": {d: bench_dataset(d, a) for d in ("modelnet", "redwood", "3dmatch")},
            "cloud_subsample_8_clouds_N10240": bench_subsample(a)}
    print(json.dumps(line))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
