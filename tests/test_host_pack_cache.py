"""CPU: bookkeeping of the packed tensor-core weight cache (engine._tc_workspace / prepack_weights) -- which calls see
`already packed`, what invalidates an entry, which entries a one-launch re-pack would pick.  No kernel runs here."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _weight(cout=64, cin=32):
    return torch.nn.Parameter(torch.randn(cout, cin, 1))     # a Conv1d(k=1) weight


def test_workspace_reuse_and_invalidation():
    from usip_b200 import _lib, engine
    p = _weight()
    ws, packed, ent = engine._tc_workspace(p, 0, 4096, 32, 64, False)
    assert not packed and ws.numel() == 2 * 32 * 64 and ent is not None
    ws2, packed2, ent2 = engine._tc_workspace(p, 0, 4096, 32, 64, False)
    assert packed2 and ws2 is ws and ent2 is ent            # same shape, same weights: reuse
    _, packed3, ent3 = engine._tc_workspace(p, 0, 4096, 32, 64, True)
    assert not packed3 and ent3 is not ent                  # the transposed (dgrad) use packs its own tiles
    with torch.no_grad():
        p.add_(1.0)                                         # autograd version bump (what an eager optimizer does)
    _, packed4, ent4 = engine._tc_workspace(p, 0, 4096, 32, 64, False)
    assert not packed4 and ent4 is ent and ent4.ws is ws    # stale: same workspace, packed again
    _lib.WEIGHT_GEN[0] += 1                                 # what usip_adam_step / a graph replay do
    _, packed5, _ = engine._tc_workspace(p, 0, 4096, 32, 64, False)
    assert not packed5
    engine.invalidate_packed_weights(torch.nn.ParameterList([p]))
    _, packed6, ent6 = engine._tc_workspace(p, 0, 4096, 32, 64, False)
    assert not packed6 and ent6 is not ent                  # cache dropped


def test_concat_halves_get_separate_entries():
    from usip_b200 import engine
    p = _weight(64, 96)                                     # a layer on cat(a [.., 64], b [.., 32])
    ws_a, _, ea = engine._tc_workspace(p, 0, 4096, 64, 64, False)
    ws_b, packed_b, eb = engine._tc_workspace(p, 64, 4096, 32, 64, False)
    assert not packed_b and eb is not ea and ws_b is not ws_a and ws_b.numel() == 2 * 32 * 64
    _, packed_a, ea2 = engine._tc_workspace(p, 0, 4096, 64, 64, False)
    _, packed_b2, eb2 = engine._tc_workspace(p, 64, 4096, 32, 64, False)
    assert packed_a and ea2 is ea and packed_b2 and eb2 is eb


def test_prepack_selects_only_stale_entries_used_by_the_last_step():
    from usip_b200 import _lib, engine

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.a = _weight()
            self.b = _weight()
    net = Net()
    assert engine.prepack_weights(net) == 0                 # nothing registered yet
    _, _, ea = engine._tc_workspace(net.a, 0, 4096, 32, 64, False)
    _, _, eb = engine._tc_workspace(net.b, 0, 4096, 32, 64, False)
    # entries without a remembered descriptor (the layer never ran) are left to their own first launch
    _lib.WEIGHT_GEN[0] += 1
    assert engine.prepack_weights(net) == 0
    assert ea.desc is None and eb.desc is None
    # a fresh entry is not picked either
    step = engine._PACK_STEP[0]
    engine._tc_workspace(net.a, 0, 4096, 32, 64, False)
    assert ea.used_step == step and ea.ver == (net.a._version, _lib.WEIGHT_GEN[0])
