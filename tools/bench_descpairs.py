"""Cost of building descriptor training batches (usip_b200.data.kitti_descriptor_loader) -- one JSON line.

  * builder: ms per batch of B pairs in device mode (CUDA events), split into subsample / candidate gather + FPS /
    augment;
  * frozen detector: ms of `run_model_siamese` on a built batch, once with the packed tensor-core weights current and
    once re-packed before every call, as happens in training (`FlatAdam.step` of the descriptor bumps the global
    weight generation);
  * training loop: `ModelDescriptor.optimize()` fed from KittiDescriptorPairSource against optimize() on one resident
    batch, in the same job;
  * reference: ms per pair of the reference's KittiDescriptorLoader.__getitem__ on the host cores (only where the
    reference's Python tree is importable; otherwise "not measured").

    python tools/bench_descpairs.py [--pairs 8] [--scan-rows 20480] [--N 16384] [--M 256] [--iters 50] [--out FILE]
    python tools/bench_descpairs.py --reference-only      # host timing of the reference loader alone
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
from usip_b200 import _lib, ops  # noqa: E402
from usip_b200.data import kitti_descriptor_loader as kdesc  # noqa: E402
from usip_b200.data import kitti_detector_loader as kdl  # noqa: E402


def desc_opt(N, M, B, device):
    from tests.util_gpu import make_opt
    return make_opt(input_pc_num=N, node_num=M, batch_size=B, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                    rot_perturbation=False, translation_perturbation=False, positive_radius_threshold=5.0,
                    negative_radius_threshold=50.0, ball_radius=2.0, ball_nsamples=64, node_knn_k_1=16,
                    device=device)


def trajectory(counts, spacing=1.5):
    return [[np.block([[np.eye(3), np.array([[1000.0 * s], [0.0], [spacing * i]])], [np.zeros((1, 3)), np.ones((1, 1))]])
             for i in range(n)] for s, n in enumerate(counts)]


def frozen_detector(opt):
    from oracle import usip_oracle as orc
    from tests.util_gpu import load_params
    from usip_b200.models.keypoint_detector import ModelDetector
    det = ModelDetector(opt)
    load_params(det.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    det.freeze_model()
    return det


def bench_builder(a, dev, det):
    B, N, M, S = a.pairs, a.N, a.M, 4
    arrs = [kdl.synthetic_scan(100 + i, a.scan_rows) for i in range(2 * B)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in arrs])]).astype(np.int64)
    scans = torch.from_numpy(np.concatenate(arrs)).to(dev)
    b = kdesc.DescriptorPairBuilder(desc_opt(N, M, B, dev), "train", dev, seed=1)
    anc, pos = list(range(B)), list(range(B, 2 * B))
    for s in range(5):
        b.build(scans, off, anc, pos, step=s)
    torch.cuda.synchronize()
    res = {"batch_ms": event_ms(lambda: b.build(scans, off, anc, pos), a.iters)}
    off_d = torch.from_numpy(off).to(dev)
    soc = torch.tensor(np.stack([anc, pos], 1).ravel(), dtype=torch.int32, device=dev)
    rows, cand, start = b.last["rows"], b.last["cand"], b.last["start"]
    params = b.last["params"]
    _, nodes = ops.fps(b.last["candidates"], start, M)
    res["subsample_ms"] = event_ms(lambda: ops.cloud_subsample(scans, off_d, soc, a.scan_rows, N, b.n_cand, seed=1),
                                   a.iters)
    res["gather_fps_ms"] = event_ms(lambda: ops.fps(ops.cloud_gather_candidates(scans, off_d, soc, rows, cand), start,
                                                    M), a.iters)
    res["augment_ms"] = event_ms(lambda: ops.desc_pair_augment(scans, off_d, soc, rows, nodes, params, S, b.flags, 1,
                                                               0), a.iters)
    # frozen detector on the built clouds
    out = b.build(scans, off, anc, pos, step=0)
    fn = lambda: det.run_model_siamese((out[0], out[3]), (out[1], out[4]), (out[2], out[5]))
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    res["detector_ms"] = event_ms(fn, a.iters)

    def repacked():
        _lib.WEIGHT_GEN[0] += 1
        fn()
    res["detector_repacked_ms"] = event_ms(repacked, a.iters)
    res["detector_repack_cost_ms"] = res["detector_repacked_ms"] - res["detector_ms"]
    return res


def bench_training_loop(a, dev, det):
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    B, N, M = a.pairs, a.N, a.M
    opt = desc_opt(N, M, B, dev)
    counts = [B * a.loop_batches] + [0] * 10
    with tempfile.TemporaryDirectory() as root:
        kdl.write_synthetic_kitti(root, counts, a.scan_rows, seed=5, poses=trajectory(counts))
        src = kdesc.KittiDescriptorPairSource(root, "train", opt, det, dev, seed=2)
        torch.manual_seed(0)
        md = ModelDescriptor(opt)
        for _ in range(2):                                        # warm-up: allocator, kernel attributes
            for _ in src.feed(md):
                md.optimize(epoch=0)
        torch.cuda.synchronize()
        steps, t0 = 0, time.perf_counter()
        for _ in range(a.loop_epochs):
            for _ in src.feed(md):
                md.optimize(epoch=0)
                steps += 1
        torch.cuda.synchronize()
        fed = (time.perf_counter() - t0) * 1e3 / steps
        batch = next(src.feed(md))
        md.set_input(*[t.clone() for t in batch])
        for _ in range(3):
            md.optimize(epoch=0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            md.optimize(epoch=0)
        torch.cuda.synchronize()
        resident = (time.perf_counter() - t0) * 1e3 / steps
    return {"steps": steps, "fed_step_ms": fed, "resident_step_ms": resident}


def bench_reference(a):
    """KittiDescriptorLoader.__getitem__ of the reference on the host, from a synthetic tree with a trajectory."""
    try:
        import importlib
        from oracle import ref_shim
        if not ref_shim.reference_available():
            return None
        ref_shim.install(use_ref_ext=False)
        kl = importlib.import_module("data.kitti_descriptor_loader")
    except Exception as e:                                          # the reference tree is optional
        print("[bench_descpairs] reference loader not importable: %s" % e, file=sys.stderr)
        return None
    import random
    opt = ref_shim.make_opt(input_pc_num=a.N, node_num=a.M, surface_normal_len=4, rot_horizontal=True,
                            translation_perturbation=False, rot_perturbation=False, positive_radius_threshold=5.0,
                            negative_radius_threshold=50.0)
    counts = [a.ref_items + 4] + [0] * 10
    with tempfile.TemporaryDirectory() as root:
        kdl.write_synthetic_kitti(root, counts, a.scan_rows, seed=5, poses=trajectory(counts))
        loader = kl.KittiDescriptorLoader(root, "train", opt)
        np.random.seed(0)
        random.seed(0)
        loader[0]
        t0 = time.perf_counter()
        for i in range(a.ref_items):
            loader[i]
        ms = (time.perf_counter() - t0) * 1e3 / a.ref_items
    return {"ms_per_pair": ms, "items": a.ref_items, "torch_threads": torch.get_num_threads(), "host_cpus": os.cpu_count()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--pairs", type=int, default=8)
    p.add_argument("--scan-rows", type=int, default=20480)
    p.add_argument("--N", type=int, default=16384)
    p.add_argument("--M", type=int, default=256)
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--loop-batches", type=int, default=4)
    p.add_argument("--loop-epochs", type=int, default=5)
    p.add_argument("--ref-items", type=int, default=4)
    p.add_argument("--reference-only", action="store_true")
    p.add_argument("--out", default=None)
    a = p.parse_args()
    res = {"pairs": a.pairs, "scan_rows": a.scan_rows, "N": a.N, "M": a.M}
    if not a.reference_only:
        if not torch.cuda.is_available():
            raise SystemExit("bench_descpairs needs a CUDA device")
        dev = torch.device("cuda:0")
        res["gpu"] = gpu_info()
        det = frozen_detector(desc_opt(a.N, a.M, a.pairs, dev))
        res["builder"] = bench_builder(a, dev, det)
        res["training_loop"] = bench_training_loop(a, dev, det)
    ref = bench_reference(a)
    res["reference_loader"] = ref if ref is not None else "not measured"
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
