#!/usr/bin/env python
"""Times the eight forward launches of the wgmma layer kernel (csrc/mlp_tc.cu) that dominate the detector fwd+loss step,
each standalone at the step's shapes and flags (KITTI detector, 8 pairs = 16 clouds, N = 16384, M = 512, node kNN
k = 16: P = 262144 point rows, G = 131072 node-neighbour rows), with CUDA events over many back-to-back launches.

Per layer it prints the time per launch, the achieved bandwidth against the compulsory HBM bytes (X read once, Y and the
group max/min written once) and the issued-TF32 fraction: 3 TF32 MACs per algorithmic MAC (3xTF32) against
1,024 TF32 MAC/clk/SM x SMs x the SM clock, at the clock sampled during the timed launches and at the maximum clock.

    python tools/bench_layer_tc.py [--iters N] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from usip_b200 import ops  # noqa: E402

HBM_TBS = 3.35                 # H100 SXM data sheet
TF32_MAC_PER_CLK_SM = 1024     # dense TF32 wgmma rate per SM

GRAPH_LAUNCHES = 20            # launches of one layer per captured graph
P, Q, KN = 16 * 16384, 16 * 512, 16
G = Q * KN

# name, rows, Cin, Cout, BN statistics, input affine + ReLU, addend, group max/min, Y written
LAYERS = [
    ("pn1.1", P, 64, 64, True, True, None, 0, True),
    ("pn1.2", P, 64, 64, False, True, None, 0, True),
    ("pn2.0", P, 64, 128, True, False, "index", 0, True),
    ("pn2.1", P, 128, 128, False, True, None, 0, True),
    ("knn_b1", G, 256, 256, True, True, None, 0, True),
    ("knn_b2", G, 256, 256, True, True, None, KN, True),
    ("knn_a0", G, 256, 512, True, True, "group", 0, True),
    ("knn_a1", G, 512, 512, True, True, None, KN, False),
]


def _smi(query):
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return r.stdout.strip()


def _setup(name, rows, cin, cout, stats, aff, addend, group, write_y, dev, rng):
    t = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32)).to(dev)
    kw = dict(X=t(rows, cin), W=t(cout, cin) / np.sqrt(cin), bias=t(cout), P=rows, Cin=cin, Cout=cout, precision=1)
    kw["tc_ws"] = torch.empty(2 * cin * cout, dtype=torch.float32, device=dev)
    if aff:
        kw.update(in_scale=t(cin).abs(), in_shift=t(cin), in_relu=True)
    if stats:
        kw["stat_partial"] = torch.empty((ops.stat_slots(rows, cout, 1, group, bool(group)), 2, cout), device=dev)
    if addend == "index":             # pn2.0: per-node term, row -> node through an index (cluster of the point)
        kw.update(addend=t(Q, cout), add_index=torch.from_numpy(rng.integers(0, Q, rows, dtype=np.int32)).to(dev))
    elif addend == "group":           # knn_a0: per-node term, row -> row / k
        kw.update(addend=t(Q, cout), add_group=KN)
    if group:
        kw.update(gmax=torch.empty((rows // group, cout), device=dev), gmin=torch.empty((rows // group, cout), device=dev),
                  group=group)
    if write_y:
        kw["Y"] = torch.empty((rows, cout), device=dev)
    ops.layer_fwd(**kw)               # packs the weights into tc_ws
    kw["tc_packed"] = True
    nbytes = 4.0 * rows * cin + (4.0 * rows * cout if write_y else 0.0) + (8.0 * rows // group * cout if group else 0.0)
    return kw, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=0, help="launches per layer (default: about 0.5 s of work)")
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_layer_tc: needs a CUDA GPU")
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    gpu = _smi("name,power.limit,clocks.max.sm")
    max_mhz = float(gpu.split(",")[-1])
    res = []
    for name, rows, cin, cout, stats, aff, addend, group, write_y in LAYERS:
        kw, nbytes = _setup(name, rows, cin, cout, stats, aff, addend, group, write_y, dev, rng)
        # launches replayed from a CUDA graph (as in the step), so that host time per call does not enter the timing
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(5):
                ops.layer_fwd(**kw)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(GRAPH_LAUNCHES):
                ops.layer_fwd(**kw)
        for _ in range(3):
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
        reps = max(1, a.iters // GRAPH_LAUNCHES) if a.iters else max(10, int(500.0 / max(e0.elapsed_time(e1), 1e-3)))
        iters = reps * GRAPH_LAUNCHES
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        mhz = float(_smi("clocks.sm"))  # sampled while the enqueued launches run
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        del g
        macs = float(rows) * cin * cout
        peak = lambda f: TF32_MAC_PER_CLK_SM * sms * f * 1e6
        r = dict(layer=name, shape="%dx%d->%d" % (rows, cin, cout), ms=round(ms, 5), iters=iters,
                 hbm_bytes=int(nbytes), achieved_TBs=round(nbytes / (ms * 1e-3) / 1e12, 3),
                 hbm_floor_ms=round(nbytes / (HBM_TBS * 1e12) * 1e3, 4),
                 sm_mhz=mhz, issued_tf32_frac=round(3 * macs / (ms * 1e-3) / peak(mhz), 3),
                 issued_tf32_frac_at_max_clock=round(3 * macs / (ms * 1e-3) / peak(max_mhz), 3))
        res.append(r)
        print("%-7s %-18s %8.4f ms  %5.2f TB/s  tf32 issued %.2f at %4.0f MHz (%.2f at %4.0f)"
              % (name, r["shape"], ms, r["achieved_TBs"], r["issued_tf32_frac"], mhz,
                 r["issued_tf32_frac_at_max_clock"], max_mhz), flush=True)
        del kw
    out = {"gpu": "name, power.limit, clocks.max.sm: " + gpu, "sms": sms, "layers": res,
           "total_ms": round(sum(r["ms"] for r in res), 4)}
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
