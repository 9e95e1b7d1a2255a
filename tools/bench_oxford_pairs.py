"""Cost of building Oxford training batches (usip_b200.data.oxford_detector_loader, .oxford_descriptor_loader) -- one
JSON line.

  * detector builder: ms per batch in device mode (CUDA events), split into subsample / candidate gather + FPS /
    augment, at the Oxford detector defaults (2 pairs, N=16384, M=512);
  * descriptor builder: the same at BASELINE configs[3] (8 pairs, N=16384, M=1024), and the frozen detector pass on
    the built clouds;
  * training loops: ModelDetector.optimize() fed from OxfordPairSource and ModelDescriptor.optimize() fed from
    OxfordDescriptorPairSource, each against optimize() on one resident batch, in the same job;
  * reference: ms per pair of the reference's OxfordLoader / OxfordDescriptorLoader.__getitem__ on the host cores (only
    where the reference's Python tree is importable; otherwise "not measured").
Scans are synthetic ENU scans of --scan-rows rows (write_synthetic_oxford).

    python tools/bench_oxford_pairs.py [--scan-rows 20480] [--iters 50] [--out FILE]
    python tools/bench_oxford_pairs.py --reference-only      # host timing of the reference loaders alone
"""
import argparse
import json
import os
import random
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_pairgen import event_ms, gpu_info  # noqa: E402
from usip_b200 import ops  # noqa: E402
from usip_b200.data import oxford_descriptor_loader as odesc  # noqa: E402
from usip_b200.data import oxford_detector_loader as odet  # noqa: E402

DET = (2, 16384, 512)                            # pairs, N, M: oxford/options_detector.py
DESC = (8, 16384, 1024)                          # BASELINE configs[3]


def oxford_opt(N, M, B, device, **kw):
    """oxford/options_*.py: S=4, rot_horizontal, height scaling; the descriptor's ball query r=1.0, Kb=64."""
    from tests.util_gpu import make_opt
    return make_opt(input_pc_num=N, node_num=M, batch_size=B, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                    rot_perturbation=False, translation_perturbation=False, is_height_scaling=True, ball_radius=1.0,
                    ball_nsamples=64, device=device, **kw)


def frozen_detector(opt):
    from oracle import usip_oracle as orc
    from tests.util_gpu import load_params
    from usip_b200.models.keypoint_detector import ModelDetector
    det = ModelDetector(opt)
    load_params(det.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    det.freeze_model()
    return det


def bench_builder(a, dev, desc, det=None):
    B, N, M = DESC if desc else DET
    arrs = [odet.synthetic_enu_scan(100 + i, a.scan_rows) for i in range(2 * B)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in arrs])]).astype(np.int64)
    scans = torch.from_numpy(np.concatenate(arrs)).to(dev)
    opt = oxford_opt(N, M, B, dev)
    if desc:
        b = odesc.OxfordDescriptorPairBuilder(opt, "train", dev, seed=1)
        anc, pos = list(range(B)), list(range(B, 2 * B))
        build = lambda step=None: b.build(scans, off, anc, pos, step=step)
        soc = np.stack([anc, pos], 1).ravel()
    else:
        b = odet.OxfordPairBuilder(opt, "train", dev, seed=1)
        build = lambda step=None: b.build(scans, off, list(range(B)), step=step)
        soc = np.repeat(np.arange(B), 2)
    for s in range(5):
        build(s)
    torch.cuda.synchronize()
    res = {"pairs": B, "N": N, "M": M, "batch_ms": event_ms(build, a.iters)}
    off_d = torch.from_numpy(off).to(dev)
    soc = torch.from_numpy(soc.astype(np.int32)).to(dev)
    rows, cand, start, params = (b.last[k] for k in ("rows", "cand", "start", "params"))
    zs = b._z_scale(params.cpu().numpy())
    zs = None if zs is None else torch.from_numpy(zs).to(dev)
    _, nodes = ops.fps(b.last["candidates"], start, M)
    res["subsample_ms"] = event_ms(lambda: ops.cloud_subsample(scans, off_d, soc, a.scan_rows, N, b.n_cand, seed=1),
                                   a.iters)
    res["gather_fps_ms"] = event_ms(lambda: ops.fps(ops.cloud_gather_candidates(scans, off_d, soc, rows, cand, zs),
                                                    start, M), a.iters)
    if desc:
        aug = lambda: ops.desc_pair_augment(scans, off_d, soc, rows, nodes, params, 4, b.flags, 1, 0)
    else:
        aug = lambda: ops.pair_augment(scans, off_d, soc, rows, nodes, params, 4, b.flags, 1, 0)
    res["augment_ms"] = event_ms(aug, a.iters)
    if desc:
        out = build(0)
        fn = lambda: det.run_model_siamese((out[0], out[3]), (out[1], out[4]), (out[2], out[5]))
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        res["detector_ms"] = event_ms(fn, a.iters)
        kp = fn()[0]
        res["height_scale_ms"] = event_ms(lambda: odesc.scale_height_(0.7, out[0], kp[0], out[3], kp[1]), a.iters)
    return res


def _timed_loop(src, md, epochs, seed_np=False):
    for _ in range(2):                                        # warm-up: graph capture, allocator
        for _ in src.feed(md):
            md.optimize(epoch=0)
    torch.cuda.synchronize()
    steps, t0 = 0, time.perf_counter()
    for _ in range(epochs):
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
    return {"steps": steps, "fed_step_ms": fed, "resident_step_ms": (time.perf_counter() - t0) * 1e3 / steps}


def bench_training_loops(a, dev, det):
    from oracle import usip_oracle as orc
    from tests.util_gpu import load_params
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    from usip_b200.models.keypoint_detector import ModelDetector
    res = {}
    with tempfile.TemporaryDirectory() as root:
        B, N, M = DET
        odet.write_synthetic_oxford(root, B * a.loop_batches, a.scan_rows, seed=5)
        src = odet.OxfordPairSource(root, "train", oxford_opt(N, M, B, dev), dev, seed=2)
        md = ModelDetector(oxford_opt(N, M, B, dev))
        load_params(md.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
        res["detector"] = _timed_loop(src, md, a.loop_epochs)
    with tempfile.TemporaryDirectory() as root:
        B, N, M = DESC
        odet.write_synthetic_oxford(root, B * a.loop_batches, a.scan_rows, seed=6)
        src = odesc.OxfordDescriptorPairSource(root, "train", oxford_opt(N, M, B, dev), det, dev, seed=2)
        torch.manual_seed(0)
        md = ModelDescriptor(oxford_opt(N, M, B, dev))
        res["descriptor"] = _timed_loop(src, md, a.loop_epochs)
    return res


def bench_reference(a):
    """OxfordLoader / OxfordDescriptorLoader.__getitem__ of the reference on the host, from a synthetic tree."""
    try:
        import importlib
        from oracle import ref_shim
        if not ref_shim.reference_available():
            return None
        ref_shim.install(use_ref_ext=False)
        if "torch._six" not in sys.modules:                # removed from torch; the loader only imports these names
            sys.modules["torch._six"] = types.ModuleType("torch._six")
            sys.modules["torch._six"].__dict__.update(string_classes=str, int_classes=int,
                                                     FileNotFoundError=FileNotFoundError)
        dl = importlib.import_module("data.oxford_detector_loader")
        ddl = importlib.import_module("data.oxford_descriptor_loader")
    except Exception as e:                                          # the reference tree is optional
        print("[bench_oxford_pairs] reference loaders not importable: %s" % e, file=sys.stderr)
        return None
    res = {}
    with tempfile.TemporaryDirectory() as root:
        odet.write_synthetic_oxford(root, a.ref_items + 4, a.scan_rows, seed=5)
        for name, cls, (_, N, M) in (("detector", dl.OxfordLoader, DET), ("descriptor", ddl.OxfordDescriptorLoader, DESC)):
            from oracle.ref_shim import make_opt
            loader = cls(root, "train", make_opt(input_pc_num=N, node_num=M, surface_normal_len=4, rot_horizontal=True,
                                                 rot_3d=False, rot_perturbation=False, translation_perturbation=False,
                                                 is_height_scaling=True))
            np.random.seed(0)
            random.seed(0)
            loader[0]
            t0 = time.perf_counter()
            for i in range(a.ref_items):
                loader[i]
            res[name] = {"N": N, "M": M, "ms_per_pair": (time.perf_counter() - t0) * 1e3 / a.ref_items}
    res.update(items=a.ref_items, torch_threads=torch.get_num_threads(), host_cpus=os.cpu_count())
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--scan-rows", type=int, default=20480)
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--loop-batches", type=int, default=3)
    p.add_argument("--loop-epochs", type=int, default=3)
    p.add_argument("--ref-items", type=int, default=3)
    p.add_argument("--reference-only", action="store_true")
    p.add_argument("--out", default=None)
    a = p.parse_args()
    res = {"scan_rows": a.scan_rows}
    if not a.reference_only:
        if not torch.cuda.is_available():
            raise SystemExit("bench_oxford_pairs needs a CUDA device")
        dev = torch.device("cuda:0")
        res["gpu"] = gpu_info()
        det = frozen_detector(oxford_opt(DESC[1], DESC[2], DESC[0], dev))
        res["detector_builder"] = bench_builder(a, dev, False)
        res["descriptor_builder"] = bench_builder(a, dev, True, det)
        res["training_loop"] = bench_training_loops(a, dev, det)
    ref = bench_reference(a)
    res["reference_loader"] = ref if ref is not None else "not measured"
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
