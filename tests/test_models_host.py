"""CPU: the model layer's contracts -- each network is built like the reference's (same state_dict keys, order and initial
values under one torch seed, same parameter order), the input staging of all three models, and the CPU-device behaviour
of the two descriptor models."""
import contextlib
import os
import subprocess
import sys
import types

import pytest
import torch

from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 7
NETWORKS = {"RPN_Detector": {}, "RPN_DetectorLite": {}, "RPN_Detector_KNN": {}, "RPN_Detector_Ball": {},
            "DescriptorLiteOld": {}, "DescriptorLiteOldGlobal": dict(ball_nsamples=448)}

# Builds the reference networks in a process of their own: the cpu-mode shim patches torch.cuda for the whole process.
_REFERENCE_BUILD = """
import importlib, sys, torch
sys.path.insert(0, sys.argv[1])
from oracle import ref_shim
from tests.test_models_host import NETWORKS, SEED
ref_shim.install(mode="cpu")
networks = importlib.import_module("models.networks")
out = {}
for name, over in NETWORKS.items():
    torch.manual_seed(SEED)
    net = getattr(networks, name)(ref_shim.make_opt(**over))
    out[name] = (net.state_dict(), [n for n, _ in net.named_parameters()])
torch.save(out, sys.argv[2])
"""


@pytest.fixture(scope="module")
def reference_networks(tmp_path_factory):
    if not ref_shim.reference_available():
        pytest.skip("the reference tree is neither mounted nor staged under oracle/_ref/py")
    path = str(tmp_path_factory.mktemp("ref") / "networks.pt")
    r = subprocess.run([sys.executable, "-c", _REFERENCE_BUILD, ROOT, path], capture_output=True, text=True, cwd=ROOT,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return torch.load(path)


@pytest.mark.parametrize("name", list(NETWORKS))
def test_network_construction_matches_the_reference(name, reference_networks):
    """Same submodules created in the same order: the torch RNG draws, the state_dict and the parameter order
    (which FlatAdam and the backward plans flatten) all follow from it."""
    from usip_b200.models import networks
    torch.manual_seed(SEED)
    net = getattr(networks, name)(ref_shim.make_opt(**NETWORKS[name]))
    ref_sd, ref_params = reference_networks[name]
    sd = net.state_dict()
    assert list(sd) == list(ref_sd)
    for k, v in ref_sd.items():
        assert sd[k].dtype == v.dtype and torch.equal(sd[k], v), k
    assert [n for n, _ in net.named_parameters()] == ref_params


def _models():
    from usip_b200.models.keypoint_descriptor import ModelDescriptor, ModelDescriptorIndoor
    from usip_b200.models.keypoint_detector import ModelDetector
    return {"ModelDetector": ModelDetector, "ModelDescriptor": ModelDescriptor,
            "ModelDescriptorIndoor": ModelDescriptorIndoor}


@pytest.fixture
def fake_cuda(monkeypatch):
    """torch.cuda's stream, event and synchronise calls as recorders, so that staging runs without a device."""
    calls = types.SimpleNamespace(waited=[], syncs=0)

    class _Stream:
        def __init__(self, *a, **k):
            pass

        def wait_event(self, ev):
            calls.waited.append(ev)

    class _Event:
        def record(self, stream=None):
            pass

    def _sync(*a, **k):
        calls.syncs += 1

    monkeypatch.setattr(torch.cuda, "Stream", _Stream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: _Stream())
    monkeypatch.setattr(torch.cuda, "synchronize", _sync)
    monkeypatch.setattr(torch.Tensor, "record_stream", lambda self, s: None)
    calls.Event = _Event
    return calls


@pytest.mark.parametrize("model", ["ModelDetector", "ModelDescriptor", "ModelDescriptorIndoor"])
def test_staging_contract(model, fake_cuda):
    cls = _models()[model]
    md = cls.__new__(cls)
    md.opt = types.SimpleNamespace(device=torch.device("cpu"))
    fields = cls._INPUT_FIELDS
    # float64 batches (neg_idx int32): staging stores float32, and int64 for the index field
    args = tuple(torch.tensor([1, 0], dtype=torch.int32) if k == "neg_idx" else torch.rand(2, 3, 5, dtype=torch.float64)
                 for k in fields)

    def check():
        for k, a in zip(fields, args):
            v = getattr(md, k)
            assert v.dtype == (torch.int64 if k == "neg_idx" else torch.float32), k
            assert torch.equal(v, a.to(v.dtype)), k

    done = fake_cuda.Event()
    md.prefetch_input(*args, after=done)
    assert fake_cuda.waited[-1] is done
    md.set_input(*args)                                      # adopts the staged copies: a stream wait, no synchronise
    assert fake_cuda.syncs == 0 and md._staged is None
    check()
    for k in fields:
        setattr(md, k, None)
    md.set_input(*args)                                      # nothing staged: copy, then synchronise
    assert fake_cuda.syncs == 1
    check()
    with pytest.raises(TypeError, match="set_input tensors"):
        md.prefetch_input(*args[:-1])


def test_descriptor_models_on_a_cpu_device():
    from usip_b200.models.keypoint_descriptor import ModelDescriptor, ModelDescriptorIndoor
    opt = lambda **k: ref_shim.make_opt(gpu_ids=[0], device=torch.device("cpu"), batch_size=1, input_pc_num=64,
                                        node_num=8, **k)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ModelDescriptor(opt())                               # FlatAdam takes CUDA parameters only
    md = ModelDescriptorIndoor(opt(ball_nsamples=448, descriptor_len=64, CGF_radius=0.075))
    assert md.optimizer_descriptor is None                   # constructs for state_dict work, but does not train
    for step in (md.optimize, md.test_model):
        with pytest.raises(NotImplementedError, match="DescCGFLoss"):
            step()
    for cls in (ModelDescriptor, ModelDescriptorIndoor):
        with pytest.raises(RuntimeError, match="needs a CUDA device"):
            cls(ref_shim.make_opt(gpu_ids=[-1]))
