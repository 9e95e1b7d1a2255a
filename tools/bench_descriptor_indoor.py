#!/usr/bin/env python
"""The indoor descriptor (DescriptorLiteOldGlobal: N=10240, M=512 keypoints, 448-sample balls of radius 0.75, S=4,
D=128) on synthetic clouds, eval BatchNorm, batches of 1, 4 and 8 clouds:

  * ModelDescriptorIndoor.run_model per batch (device events around work that ends in a synchronise) and clouds/s;
  * per-op device times of one profiled run_model per batch size (engine.collect_profile, a separate pass);
  * the unmodified reference network on the same GPU (its ball_query extension behind tests/desc_indoor_ref.py's
    ball_query_wrapper), when oracle/_ref holds it;
  * IndoorRegistration.describe (detector pass + descriptor pass) in scans/s on the first scene of a synthetic Redwood
    tree of 30000-row fragments; the networks are randomly initialised.

The card's name and power limit are read in the same run.  `python tools/bench_descriptor_indoor.py --out FILE`."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import desc_indoor_ref as dref  # noqa: E402
from tools.bench_registration_indoor import card, timed  # noqa: E402
from usip_b200 import engine  # noqa: E402
from usip_b200.evaluation import indoor_registration as idr  # noqa: E402
from usip_b200.evaluation import indoor_test_loader as itl  # noqa: E402
from usip_b200.evaluation import registration as reg  # noqa: E402
from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor  # noqa: E402
from usip_b200.models.keypoint_detector import ModelDetector  # noqa: E402

N, M, K, S, D = 10240, 512, 448, 4, 128
BATCHES = (1, 4, 8)


def inputs(B):
    pc, sn, kp = dref.make_inputs(B, N, M, S, seed=B, half=1.5)
    return [torch.from_numpy(a).cuda() for a in (pc, sn, kp)]


def reference_network(state):
    from oracle import build_ref, ref_shim
    if not (ref_shim.reference_available() and build_ref.have("ball_query") and build_ref.have("index_max")):
        return None
    ref = ref_shim.modules(mode="cuda")
    dref.install(ref)
    opt = ref_shim.make_opt(ball_radius=0.75, ball_nsamples=K, descriptor_len=D, surface_normal_len=S)
    net = ref.networks.DescriptorLiteOldGlobal(opt)
    net.load_state_dict(state)
    return net.cuda().eval()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/descriptor_indoor_h100.json")
    ap.add_argument("--rows", type=int, default=30000)
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = card()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    opt = reg.descriptor_opt("redwood", input_pc_num=N, node_num=M, batch_size=8)
    torch.manual_seed(0)
    md = ModelDescriptorIndoor(opt)
    state = dref.randomized_params(md.descriptor, 0)
    md.descriptor.load_state_dict(state)
    md.freeze_model()
    out = {"workload": "ModelDescriptorIndoor.run_model, eval BN: N=%d, M=%d, K=%d, r=0.75, S=%d, D=%d" % (N, M, K, S, D),
           "gpu": name, "power_limit": power, "run_model": {}, "profile_ms": {}, "reference_gpu": {}}
    for B in BATCHES:
        x, s, k = inputs(B)
        ms, _ = timed(lambda: md.run_model(x, s, k), reps=10)
        out["run_model"][str(B)] = {"ms": ms, "clouds_per_s": B / (ms * 1e-3)}
    for B in BATCHES:                                          # profiled pass: events around every op, its own run
        x, s, k = inputs(B)
        engine.PROFILE = {}
        md.run_model(x, s, k)
        torch.cuda.synchronize()
        out["profile_ms"][str(B)] = {op: round(r["ms"], 4) for op, r in engine.collect_profile().items()}
        engine.PROFILE = None
    net = reference_network(state)
    if net is None:
        out["reference_gpu"] = "not measured: oracle/_ref holds no reference build"
    else:
        for B in BATCHES:
            x, s, k = inputs(B)

            def ref_fwd():
                with torch.no_grad():
                    return net(x, s, k, False, None)[0]
            ms, d_ref = timed(ref_fwd, reps=3)
            np.random.seed(0)
            d_ref = ref_fwd()
            np.random.seed(0)
            d = md.run_model(x, s, k)
            err = float((d - d_ref).abs().max() / d_ref.abs().max())
            out["reference_gpu"][str(B)] = {"ms": ms, "speedup": ms / out["run_model"][str(B)]["ms"], "rel_err": err}
        del net
        torch.cuda.empty_cache()
    # describe on a synthetic Redwood scene
    with tempfile.TemporaryDirectory(prefix="usip_desc_indoor_") as tmp:
        npy, gt = os.path.join(tmp, "npy"), os.path.join(tmp, "gt")
        scene = itl.REDWOOD_SCENES[0]
        itl.write_synthetic_redwood(npy, gt, a.rows, {scene[0]: [(0, 2)]}, seed=0, scenes=(scene,))
        det = ModelDetector(opt)
        det.freeze_model()
        ev = idr.IndoorRegistration.redwood(npy, gt, opt, scenes=[scene], batch_size=8)
        ev.describe(det, md)                                   # warm-up: file loads, first launches
        torch.cuda.synchronize()
        ms, _ = timed(lambda: ev.describe(det, md), reps=2)
    out["describe"] = {"scene": scene[0], "scans": scene[1], "rows": a.rows, "ms": ms, "scans_per_s": scene[1] / (ms * 1e-3),
                       "includes": "fragment load and subsample, detector pass, descriptor pass, selection"}
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
