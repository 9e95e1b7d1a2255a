#!/usr/bin/env python
"""The indoor descriptor's train step, ModelDescriptorIndoor.optimize(), at SceneNN's training shape (N=5000 points,
M=512 keypoints, 448-sample balls of radius 0.75, S=4, D=128, DescCGFLoss with CGF_radius 0.075, gamma 0.3, sigma_max
0.5) on synthetic pairs (tests/cgf_ref.train_inputs), batches of 2 and 8 pairs:

  * optimize() per step (device events around steps that end in a synchronise);
  * the per-op device times of one profiled step per batch (engine.collect_profile, a separate pass): the forward, the
    CGF forward / backward and the network backward by layer;
  * the unmodified reference's optimize() on the same GPU and inputs, when oracle/_ref holds it.

The card's name and power limit are read in the same run.  `python tools/bench_descriptor_indoor_train.py --out FILE`."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import cgf_ref  # noqa: E402
from tests import desc_indoor_ref as dref  # noqa: E402
from tests.util_gpu import make_opt  # noqa: E402
from tools.bench_registration_indoor import card, timed  # noqa: E402
from usip_b200 import engine  # noqa: E402
from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor  # noqa: E402

N, M, K, S, D = 5000, 512, 448, 4, 128
BATCHES = (2, 8)


def options(B):
    return make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=0.75, ball_nsamples=K,
                    descriptor_len=D, CGF_radius=0.075, triple_loss_gamma=0.3, sigma_max=0.5,
                    random_pc_dropout_lower_limit=1.0)


def batch(B):
    d = cgf_ref.train_inputs(B, N, M, S, seed=B)
    return [torch.from_numpy(d[k]) for k in cgf_ref.SET_INPUT_KEYS]


def reference_model(B, state):
    from oracle import build_ref, ref_shim
    if not (ref_shim.reference_available() and build_ref.have("ball_query") and build_ref.have("index_max")):
        return None
    ref = ref_shim.modules(mode="cuda")
    dref.install(ref)
    opt = options(B)
    md = ref.keypoint_descriptor.ModelDescriptorIndoor(ref_shim.make_opt(**{k: getattr(opt, k) for k in vars(opt)}))
    md.descriptor.load_state_dict(state)
    return md


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/descriptor_indoor_train_h100.json")
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = card()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"workload": "ModelDescriptorIndoor.optimize: N=%d, M=%d, K=%d, r=0.75, S=%d, D=%d, DescCGFLoss r=0.075" % (
        N, M, K, S, D), "gpu": name, "power_limit": power, "optimize": {}, "profile_ms": {}, "reference_gpu": {}}
    states = {}
    for B in BATCHES:
        torch.manual_seed(0)
        md = ModelDescriptorIndoor(options(B))
        states[B] = dref.randomized_params(md.descriptor, 0)
        md.descriptor.load_state_dict(states[B])
        ins = batch(B)
        md.set_input(*ins)
        np.random.seed(0)
        md.optimize(epoch=0)                                   # warm-up: first launches, packed weights
        ms, _ = timed(lambda: md.optimize(epoch=0), reps=a.steps)
        out["optimize"][str(B)] = {"ms": ms, "pairs_per_s": B / (ms * 1e-3), "loss": md.loss.item()}
        engine.PROFILE = {}                                    # profiled pass: events around every op, its own step
        md.optimize(epoch=0)
        torch.cuda.synchronize()
        out["profile_ms"][str(B)] = {op: round(r["ms"], 4) for op, r in engine.collect_profile().items()}
        engine.PROFILE = None
        del md
        torch.cuda.empty_cache()
    for B in BATCHES:
        md = reference_model(B, states[B])
        if md is None:
            out["reference_gpu"] = "not measured: oracle/_ref holds no reference build"
            break
        md.set_input(*batch(B))
        np.random.seed(0)
        md.optimize(epoch=0)
        ms, _ = timed(lambda: md.optimize(epoch=0), reps=max(2, a.steps // 3))
        out["reference_gpu"][str(B)] = {"ms": ms, "speedup": ms / out["optimize"][str(B)]["ms"]}
        del md
        torch.cuda.empty_cache()
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
