"""CPU: the indoor descriptor's host side -- the restated ball_query_wrapper the reference network needs, the reference
network against tests/golden/descriptor_indoor.npz, DescriptorLiteOldGlobal's state_dict and refusals,
ModelDescriptorIndoor's forward-only surface, and the indoor registration CLI's choice of descriptor model."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import ref_shim, usip_oracle as orc
from tests import desc_indoor_ref as dref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "descriptor_indoor.npz")


def _opt(**over):
    o = ref_shim.make_opt(gpu_ids=[0], ball_radius=0.75, ball_nsamples=448, descriptor_len=128.0, surface_normal_len=4)
    o.__dict__.update(over)
    return o


def _balls(K):
    """Three keypoints per cloud: an empty ball, a partly filled one (fewer than K hits) and an over-full one."""
    rng = np.random.default_rng(K)
    B, N = 2, 3000
    pc = rng.uniform(-1, 1, (B, 3, N)).astype(np.float32)
    pc[:, :, : 2 * K] = rng.uniform(-0.2, 0.2, (B, 3, 2 * K))            # a dense core: over-full at the centre
    kp = np.zeros((B, 3, 3), np.float32)
    kp[:, :, 0] = 40.0
    kp[:, :, 1] = 0.97                                                   # a cube corner: partly filled
    return pc, kp


@pytest.mark.parametrize("K", [448, 64])
def test_ball_query_wrapper_restatement(K, monkeypatch):
    """The shim's ball_query_wrapper (distance matrix by torch.norm, then the ball query the cpu-mode shim installs)
    against the oracle's ball query and against the commented-out numba kernel it restates."""
    monkeypatch.setitem(sys.modules, "ball_query", types.SimpleNamespace(
        forward_cuda_shared_mem=ref_shim._ball_query_restatement))
    pc, kp = _balls(K)
    r = 0.75 if K == 448 else 0.3
    got = dref.ball_query_wrapper(torch.from_numpy(pc), torch.from_numpy(kp), r, K)
    assert got.dtype == torch.int64 and tuple(got.shape) == (2, 3, K)
    dist = torch.norm(torch.from_numpy(kp).unsqueeze(3) - torch.from_numpy(pc).unsqueeze(2), p=2, dim=1).numpy()
    hits = (dist <= np.float32(r)).sum(2)
    assert (hits[:, 0] == 0).all() and ((hits[:, 1] > 0) & (hits[:, 1] < K)).all() and (hits[:, 2] > K).all(), hits
    want = orc.ball_query_dist(np.ascontiguousarray(dist), r, K)
    np.testing.assert_array_equal(got.numpy(), want)
    np.testing.assert_array_equal(dref.numba_ball_query(dist, r, K), want)
    assert (got[:, 0] == 0).all()                                        # empty ball: index 0


def test_reference_network_reproduces_golden():
    """The unmodified reference DescriptorLiteOldGlobal on the CPU through the shim (its own process: the cpu-mode shim
    patches torch.cuda) reproduces the golden file."""
    if not ref_shim.reference_available():
        pytest.skip("the reference tree is neither mounted nor staged under oracle/_ref/py")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "desc_indoor_ref.py"), GOLDEN], capture_output=True,
                       text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    vals = dict(line.split() for line in r.stdout.splitlines() if line.strip())
    assert float(vals["desc_eval"]) <= 1e-5 and float(vals["desc_train"]) <= 1e-5, vals
    assert vals["feats_eval"] == "0" and vals["feats_train"] == "0", vals
    stats = {k: float(v) for k, v in vals.items() if k.startswith("after/")}
    assert len(stats) == 18 and max(stats.values()) <= 1e-6, stats


def _expected_shapes(D, cin=7):
    shapes = {}
    for name, (o, i) in dict(conv1=(D // 4, cin), conv2=(D // 2, D // 4), conv3=(D, D // 2), conv4=(D, 2 * D),
                             conv5=(D, D)).items():
        shapes[name + ".conv.weight"], shapes[name + ".conv.bias"] = (o, i, 1, 1), (o,)
    for name, (o, i) in dict(fc1=(2 * D, 2 * D), fc2=(D, 2 * D), fc3=(D, D)).items():
        shapes[name + ".conv.weight"], shapes[name + ".conv.bias"] = (o, i, 1), (o,)
    for name in ("conv1", "conv2", "conv3", "conv4", "fc1", "fc2"):
        o = shapes[name + ".conv.bias"]
        for k in ("weight", "bias", "running_mean", "running_var"):
            shapes["%s.norm.%s" % (name, k)] = o
        shapes[name + ".norm.num_batches_tracked"] = ()
    return shapes


def test_state_dict_matches_reference_and_loads_checkpoints(tmp_path):
    from usip_b200.evaluation.repeatability import load_checkpoint
    from usip_b200.models.networks import DescriptorLiteOldGlobal
    net = DescriptorLiteOldGlobal(_opt())                              # descriptor_len given as a float, as the options
    got = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert got == _expected_shapes(128)
    # the reference's own state_dict (golden file, D=64): same keys and shapes, loads strictly with and without module.
    g = np.load(GOLDEN)
    sd = {k[len("param/"):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("param/")}
    small = DescriptorLiteOldGlobal(_opt(descriptor_len=int(g["D"])))
    assert {k: tuple(v.shape) for k, v in small.state_dict().items()} == {k: tuple(v.shape) for k, v in sd.items()}
    for prefix in ("", "module."):
        path = str(tmp_path / ("sd%s.pth" % prefix))
        torch.save({prefix + k: v for k, v in sd.items()}, path)
        fresh = DescriptorLiteOldGlobal(_opt(descriptor_len=int(g["D"])))
        load_checkpoint(fresh, path)                                   # load_state_dict(strict=True)
        for k, v in fresh.state_dict().items():
            assert torch.equal(v, sd[k]), k
    with pytest.raises(RuntimeError):
        net.load_state_dict({k: v for k, v in net.state_dict().items() if "fc3" not in k})


def test_weight_init_follows_the_reference():
    from usip_b200.models.networks import DescriptorLiteOldGlobal
    torch.manual_seed(0)
    net = DescriptorLiteOldGlobal(_opt())
    for name in ("fc1", "fc2", "fc3", "conv4"):
        layer = getattr(net, name)
        n = layer.conv.weight[0].numel()
        std = float(layer.conv.weight.detach().std())
        assert abs(std - (2.0 / n) ** 0.5) < 0.1 * (2.0 / n) ** 0.5, (name, std)
        assert float(layer.conv.bias.abs().max()) == 0.0
    assert float(net.fc1.norm.weight.min()) == 1.0 and float(net.fc1.norm.bias.abs().max()) == 0.0


def test_ball_sizes_and_refusals(monkeypatch):
    from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
    from usip_b200.models.networks import DescriptorLiteOld, DescriptorLiteOldGlobal
    for K in (448, 192, 256, 64, 32, 128):
        DescriptorLiteOldGlobal(_opt(ball_nsamples=K))
    for K in (100, 96, 200, 130):
        with pytest.raises(NotImplementedError):
            DescriptorLiteOldGlobal(_opt(ball_nsamples=K))
    with pytest.raises(NotImplementedError):
        DescriptorLiteOld(_opt(ball_nsamples=448, descriptor_len=128))   # the outdoor descriptor keeps its check
    md = ModelDescriptorIndoor(_opt(device=torch.device("cpu"), batch_size=1, input_pc_num=64, node_num=8))
    with pytest.raises(NotImplementedError, match="DescCGFLoss"):
        md.optimize(epoch=0)
    with pytest.raises(NotImplementedError, match="DescCGFLoss"):
        md.test_model()
    x = torch.zeros(1, 3, 64)
    with pytest.raises(NotImplementedError, match="DescCGFLoss"):
        md.descriptor(x, torch.zeros(1, 4, 64), torch.zeros(1, 3, 8))   # grad enabled, trainable parameters
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)        # set_input ends in one; there is no device here
    md.set_input(x, torch.zeros(1, 4, 64), torch.zeros(1, 3, 8), torch.ones(1, 8), x, torch.zeros(1, 4, 64),
                 torch.zeros(1, 3, 8), torch.ones(1, 8), torch.eye(3)[None], torch.ones(1, 1), torch.zeros(1, 3, 1))
    md.freeze_model()
    assert not any(p.requires_grad for p in md.descriptor.parameters())
    with pytest.raises(RuntimeError, match="CUDA"):
        md.descriptor(x, torch.zeros(1, 4, 64), torch.zeros(1, 3, 8))   # frozen: refused for the CPU tensor only


@pytest.mark.parametrize("dataset", ["redwood", "3dmatch"])
def test_indoor_cli_builds_the_indoor_descriptor(dataset, monkeypatch, tmp_path):
    from usip_b200.evaluation import indoor_registration as idr
    from usip_b200.evaluation import registration as reg
    from usip_b200.evaluation import repeatability as rep
    from usip_b200.models import keypoint_descriptor as kd
    from usip_b200.models import keypoint_detector as kdet
    seen = {}

    class Stub:
        def __init__(self, opt):
            seen.setdefault("built", []).append((type(self).__name__, opt.ball_nsamples, opt.ball_radius))

    class ModelDetector(Stub):
        pass

    class ModelDescriptorIndoor(Stub):
        pass

    class Ev:
        def describe(self, det, des, nms_radius, L):
            seen["describe"] = (type(det).__name__, type(des).__name__, L)

        def score(self, *a):
            return types.SimpleNamespace(lines=lambda: ["ok"])

    monkeypatch.setattr(kdet, "ModelDetector", ModelDetector)
    monkeypatch.setattr(kd, "ModelDescriptorIndoor", ModelDescriptorIndoor)
    monkeypatch.setattr(kd, "ModelDescriptor", None)                   # the outdoor model must not be used
    monkeypatch.setattr(rep, "load_detector_checkpoint", lambda m, p: seen.__setitem__("det", p))
    monkeypatch.setattr(reg, "load_descriptor_checkpoint", lambda m, p: seen.__setitem__("des", (type(m).__name__, p)))
    monkeypatch.setattr(idr.IndoorRegistration, "redwood", classmethod(lambda cls, *a, **k: Ev()))
    monkeypatch.setattr(idr.IndoorRegistration, "match3d", classmethod(lambda cls, *a, **k: Ev()))
    argv = [dataset, "--root", str(tmp_path), "--detector", "d.pth", "--descriptor", "e.pth", "--keypoint-nums", "64",
            "128", "--max-trials", "1000"]
    if dataset == "redwood":
        argv += ["--gt-root", str(tmp_path)]
    idr.main(argv)
    assert seen["built"] == [("ModelDetector", 448, 0.75), ("ModelDescriptorIndoor", 448, 0.75)]
    assert seen["des"] == ("ModelDescriptorIndoor", "e.pth") and seen["det"] == "d.pth"
    assert seen["describe"] == ("ModelDetector", "ModelDescriptorIndoor", 128)
