"""Cost of building detector training pairs (usip_b200.data.kitti_detector_loader) -- one JSON line.

  * builder: ms per batch of B pairs in device mode (CUDA events), split into subsample / candidate gather + FPS /
    augment, and the augment kernel's GB/s against its compulsory bytes;
  * reference: ms per pair of the reference's KittiLoader.__getitem__ on the host cores (only where the reference's
    Python tree is importable; otherwise "not measured");
  * training loop: KittiPairSource + optimize() per step against optimize() on one resident batch.

    python tools/bench_pairgen.py [--pairs 8] [--scan-rows 20480] [--N 16384] [--M 512] [--iters 50] [--out FILE]
    python tools/bench_pairgen.py --reference-only      # host timing of the reference loader alone
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from usip_b200 import ops  # noqa: E402
from usip_b200.data import kitti_detector_loader as kdl  # noqa: E402


def kitti_opt(N, M, B, device):
    from tests.util_gpu import make_opt
    return make_opt(input_pc_num=N, node_num=M, batch_size=B, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                    rot_perturbation=False, translation_perturbation=False, radius_threshold=100.0, device=device)


def event_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def bench_builder(a, dev):
    B, N, M, S, C = a.pairs, a.N, a.M, 4, 8
    arrs = [kdl.synthetic_scan(100 + i, a.scan_rows) for i in range(B)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in arrs])]).astype(np.int64)
    scans = torch.from_numpy(np.concatenate(arrs)).to(dev)
    b = kdl.DetectorPairBuilder(kitti_opt(N, M, B, dev), "train", dev, seed=1)
    items = list(range(B))
    for s in range(5):
        b.build(scans, off, items, step=s)
    torch.cuda.synchronize()
    res = {"batch_ms": event_ms(lambda: b.build(scans, off, items), a.iters)}
    # the three stages alone, on the inputs of one build
    off_d = torch.from_numpy(off).to(dev)
    sp = torch.arange(B, dtype=torch.int32, device=dev).repeat_interleave(2)      # both clouds of pair b: scan b
    rows, cand, start = b.last["rows"], b.last["cand"], b.last["start"]
    params = b.last["params"]
    _, nodes = ops.fps(b.last["candidates"], start, M)
    res["subsample_ms"] = event_ms(lambda: ops.cloud_subsample(scans, off_d, sp, a.scan_rows, N, b.n_cand, None, 1, 0),
                                   a.iters)
    res["gather_fps_ms"] = event_ms(lambda: ops.fps(ops.cloud_gather_candidates(scans, off_d, sp, rows, cand), start,
                                                    M), a.iters)
    res["augment_ms"] = event_ms(lambda: ops.pair_augment(scans, off_d, sp, rows, nodes, params, S, b.flags, 1, 0),
                                 a.iters)
    # compulsory bytes of the augment kernel: row ids, the used scan columns and the nodes in; the nine outputs out
    nbytes = 2 * B * (N * 4 + N * (3 + S) * 4 + 3 * M * 4) + 2 * B * ((3 + S) * N + 3 * M) * 4 + B * 13 * 4
    res["augment_gbs"] = nbytes / (res["augment_ms"] * 1e-3) / 1e9
    res["augment_bytes"] = nbytes
    return res


def bench_training_loop(a, dev):
    from oracle import usip_oracle as orc
    from tests.util_gpu import load_params
    from usip_b200.models.keypoint_detector import ModelDetector
    B, N, M = a.pairs, a.N, a.M
    opt = kitti_opt(N, M, B, dev)
    with tempfile.TemporaryDirectory() as root:
        kdl.write_synthetic_kitti(root, [B * a.loop_batches] + [0] * 10, a.scan_rows, seed=5)
        src = kdl.KittiPairSource(root, "train", opt, dev, seed=2)
        md = ModelDetector(opt)
        load_params(md.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
        for _ in range(2):                                        # warm-up: graph capture, allocator
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
        batch = src.builder.build(src.scans, src.offsets, list(range(B)), step=0)
        md.set_input(*batch)
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
    """KittiLoader.__getitem__ of the reference on the host, from a staged synthetic tree (N, M as configured)."""
    try:
        import importlib
        from oracle import ref_shim
        if not ref_shim.reference_available():
            return None
        ref_shim.install(use_ref_ext=False)
        kl = importlib.import_module("data.kitti_detector_loader")
    except Exception as e:                                          # the reference tree is optional
        print("[bench_pairgen] reference loader not importable: %s" % e, file=sys.stderr)
        return None
    opt = ref_shim.make_opt(input_pc_num=a.N, node_num=a.M, surface_normal_len=4, rot_horizontal=True,
                            radius_threshold=100.0, translation_perturbation=False, rot_perturbation=False)
    with tempfile.TemporaryDirectory() as root:
        kdl.write_synthetic_kitti(root, [a.ref_items] + [0] * 10, a.scan_rows, seed=5)
        loader = kl.KittiLoader(root, "train", opt)
        np.random.seed(0)
        loader[0]
        t0 = time.perf_counter()
        for i in range(a.ref_items):
            loader[i]
        ms = (time.perf_counter() - t0) * 1e3 / a.ref_items
    return {"ms_per_pair": ms, "items": a.ref_items, "torch_threads": torch.get_num_threads(), "host_cpus": os.cpu_count()}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0] if q else None
    except Exception:
        return None


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--pairs", type=int, default=8)
    p.add_argument("--scan-rows", type=int, default=20480)
    p.add_argument("--N", type=int, default=16384)
    p.add_argument("--M", type=int, default=512)
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
            raise SystemExit("bench_pairgen needs a CUDA device")
        dev = torch.device("cuda:0")
        res["gpu"] = gpu_info()
        res["builder"] = bench_builder(a, dev)
        res["training_loop"] = bench_training_loop(a, dev)
    ref = bench_reference(a)
    res["reference_loader"] = ref if ref is not None else "not measured"
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
