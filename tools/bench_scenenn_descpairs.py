"""Cost of building SceneNN descriptor training batches (usip_b200.data.scenenn_descriptor_loader) -- one JSON line.

At SceneNN's descriptor shape (scenenn/options_descriptor.py: N=5000, M=512, S=4, 448-sample balls), for B = 2 and 8
pairs:
  * builder: ms per batch in device mode (CUDA events), split into subsample / float64 ICP'd gather + usip_fps_f64 /
    augment;
  * frozen detector: ms of `run_model_siamese` on a built batch;
  * training loop: `ModelDescriptorIndoor.optimize()` fed from SceneNNDescriptorPairSource ("train+val") against
    optimize() on one resident batch, in the same job;
  * reference: ms per pair of the reference's SceneNNDescriptorLoader.__getitem__ on the host cores (only where the
    reference's Python tree is importable; otherwise "not measured").

The fragments are synthetic, FRAG_ROWS = 30,000 rows each (every positive the rigid image of its anchor).  That size is
an assumption, not a measurement of SceneNN's frames, which are not available here; the row count only changes the
subsample's share of the build.

    python tools/bench_scenenn_descpairs.py [--pairs 2 8] [--frag-rows 30000] [--iters 50] [--out FILE]
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
from usip_b200.data import scenenn_descriptor_loader as sdl  # noqa: E402
from usip_b200.data import scenenn_detector_loader as snl  # noqa: E402

FRAG_ROWS = 30000
N, M, S = 5000, 512, 4


def scenenn_opt(B, device):
    """scenenn/options_descriptor.py's defaults."""
    from tests.util_gpu import make_opt
    return make_opt(input_pc_num=N, node_num=M, batch_size=B, surface_normal_len=S, node_knn_k_1=4, k=1,
                    rot_horizontal=True, rot_3d=False, rot_perturbation=True, translation_perturbation=False,
                    scene="indoor", ball_radius=0.75, ball_nsamples=448, descriptor_len=128, CGF_radius=0.075,
                    sigma_max=0.5, triple_loss_gamma=0.3, loss_sigma_lower_bound=1e-4, device=device)


def frozen_detector(opt):
    from oracle import usip_oracle as orc
    from tests.util_gpu import load_params
    from usip_b200.models.keypoint_detector import ModelDetector
    det = ModelDetector(opt)
    load_params(det.detector, orc.init_detector_params(S=S, seed=1, C1=64, C2=256, randomize_bn=True))  # indoor
    det.freeze_model()
    return det


def write_tree(root, n_train, n_val, rows):
    counts = {"train": 2 * n_train, "val": 2 * n_val, "test": 2}
    pairs = {"train": [(2 * k, 2 * k + 1) for k in range(n_train)], "val": [(2 * k, 2 * k + 1) for k in range(n_val)],
             "test": [(0, 1)]}
    snl.write_synthetic_scenenn(root, counts, rows, seed=5, pairs=pairs)


def bench_builder(a, B, dev, det, root):
    pairs, icp = sdl.scenenn_pairs(root, "train")
    arrs = [np.load(os.path.join(root, "frames_train", "%d.npy" % f)) for f in pairs[:B].ravel()]
    off = np.concatenate([[0], np.cumsum([len(x) for x in arrs])]).astype(np.int64)
    scans = torch.from_numpy(np.concatenate(arrs)).to(dev)
    b = sdl.SceneNNDescriptorPairBuilder(scenenn_opt(B, dev), "train", dev, seed=1)
    anc, pos, kinds = 2 * np.arange(B), 2 * np.arange(B) + 1, [ops.SCENENN_KIND_FULL] * B
    build = lambda s=None: b.build(scans, off, anc, pos, icp[:B], kinds, step=s)
    for s in range(5):
        build(s)
    torch.cuda.synchronize()
    res = {"batch_ms": event_ms(build, a.iters)}
    out = build(0)
    off_d = torch.from_numpy(off).to(dev)
    soc = torch.tensor(np.arange(2 * B), dtype=torch.int32, device=dev)
    icp_d = torch.from_numpy(np.ascontiguousarray(icp[:B])).to(dev)
    rows, cand, start, params = b.last["rows"], b.last["cand"], b.last["start"], b.last["params"]
    pts, idx = b.last["candidates"], b.last["node_idx"]
    res["subsample_ms"] = event_ms(lambda: ops.cloud_subsample(scans, off_d, soc, a.frag_rows, N, b.n_cand, seed=1),
                                   a.iters)
    res["gather_f64_fps_ms"] = event_ms(
        lambda: ops.fps_f64(ops.cloud_gather_candidates_icp_f64(scans, off_d, soc, rows, cand, icp_d), start, M),
        a.iters)
    res["augment_ms"] = event_ms(lambda: ops.scenenn_desc_pair_augment(scans, off_d, soc, rows, icp_d, pts, idx,
                                                                       params, S, b.flags), a.iters)
    fn = lambda: det.run_model_siamese((out[0], out[3]), (out[1], out[4]), (out[2], out[5]))
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    res["detector_ms"] = event_ms(fn, a.iters)
    return res


def bench_training_loop(a, B, dev, det, root):
    from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
    opt = scenenn_opt(B, dev)
    src = sdl.SceneNNDescriptorPairSource(root, "train+val", opt, det, dev, seed=2, batch_size=B)
    torch.manual_seed(0)
    md = ModelDescriptorIndoor(opt)
    for _ in src.feed(md):                                        # warm-up: allocator, kernel attributes
        md.optimize(epoch=0)
    torch.cuda.synchronize()
    steps, t0 = 0, time.perf_counter()
    for _ in range(a.loop_epochs):
        for _ in src.feed(md):
            md.optimize(epoch=0)
            steps += 1
    torch.cuda.synchronize()
    fed = (time.perf_counter() - t0) * 1e3 / steps
    md.set_input(*[t.clone() for t in next(src.feed(md))])     # no point dropout: the batch stays whole
    for _ in range(3):
        md.optimize(epoch=0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        md.optimize(epoch=0)
    torch.cuda.synchronize()
    resident = (time.perf_counter() - t0) * 1e3 / steps
    return {"steps": steps, "fed_step_ms": fed, "resident_step_ms": resident}


def bench_reference(a, root):
    """SceneNNDescriptorLoader.__getitem__ of the reference on the host, on the same synthetic tree."""
    try:
        import importlib
        from oracle import ref_shim
        if not ref_shim.reference_available():
            return None
        ref_shim.install(use_ref_ext=False)
        sl = importlib.import_module("data.scenenn_descriptor_loader")
    except Exception as e:                                          # the reference tree is optional
        print("[bench_scenenn_descpairs] reference loader not importable: %s" % e, file=sys.stderr)
        return None
    opt = ref_shim.make_opt(input_pc_num=N, node_num=M, surface_normal_len=S, rot_horizontal=True, rot_3d=False,
                            rot_perturbation=True, translation_perturbation=False)
    loader = sl.SceneNNDescriptorLoader(root, "train", opt)
    np.random.seed(0)
    loader[0]
    n = min(a.ref_items, len(loader))
    t0 = time.perf_counter()
    for i in range(n):
        loader[i]
    ms = (time.perf_counter() - t0) * 1e3 / n
    return {"ms_per_pair": ms, "items": n, "host_cpus": os.cpu_count()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--pairs", type=int, nargs="+", default=[2, 8])
    p.add_argument("--frag-rows", type=int, default=FRAG_ROWS)
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--loop-epochs", type=int, default=3)
    p.add_argument("--ref-items", type=int, default=4)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scenenn_descpairs needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"N": N, "M": M, "S": S, "frag_rows": a.frag_rows,
           "frag_rows_note": "synthetic fragments; the row count is an assumption, not SceneNN's",
           "gpu": gpu_info(), "shapes": {}}
    with tempfile.TemporaryDirectory() as root:
        B_max = max(a.pairs)
        write_tree(root, 4 * B_max, 2 * B_max, a.frag_rows)
        for B in a.pairs:
            det = frozen_detector(scenenn_opt(B, dev))
            res["shapes"]["B%d" % B] = {"builder": bench_builder(a, B, dev, det, root),
                                        "training_loop": bench_training_loop(a, B, dev, det, root)}
        ref = bench_reference(a, root)
    res["reference_loader"] = ref if ref is not None else "not measured"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
