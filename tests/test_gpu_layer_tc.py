"""-m gpu: the wgmma layer kernel (csrc/mlp_tc.cu) on shapes that stress its tiling: a single K chunk, weight panels
shorter and longer than the stage ring, row tails inside the last 64- and 128-row tile, CTAs whose two warpgroups get
unequal numbers of 64-row tiles, the group-128 combine across warpgroups, the transposed (dgrad) weight pack and the plain
TF32 precision.  Same numpy reference and tolerances as test_gpu_ops.test_layer_fwd."""
import numpy as np
import pytest
import torch

from tests.gemm_ref import tf32 as _tf32
from tests.test_gpu_ops import _layer_ref
from tests.util_gpu import cu, dev, rel_err

pytestmark = pytest.mark.gpu


def _run_case(P, Cin, Cout, group=0, transposed=False, single=False, add_group=0, seed=0):
    from usip_b200 import ops
    rng = np.random.default_rng(seed + P + 7 * Cin + Cout)
    X = rng.normal(size=(P, Cin)).astype(np.float32)
    W = (rng.normal(size=(Cout, Cin)) / np.sqrt(Cin)).astype(np.float32)
    b = rng.normal(size=Cout).astype(np.float32)
    scale = rng.normal(size=Cin).astype(np.float32); shift = rng.normal(size=Cin).astype(np.float32)
    if add_group:
        G = -(-P // add_group)
        add_idx = np.arange(P, dtype=np.int32) // add_group
    else:
        G = 37
        add_idx = rng.integers(0, G, size=P).astype(np.int32)
    addend = rng.normal(size=(G, Cout)).astype(np.float32)

    Y = torch.empty((P, Cout), device=dev())
    want_grp = bool(group)
    nt = ops.stat_slots(P, Cout, 1, group, want_grp)
    part = torch.full((nt, 2, Cout), float("nan"), device=dev())         # every slot must be written
    kw = {}
    if want_grp:
        assert P % group == 0
        Q = P // group
        kw = dict(gmax=torch.empty((Q, Cout), device=dev()), gmin=torch.empty((Q, Cout), device=dev()),
                  garg_max=torch.empty((Q, Cout), dtype=torch.int32, device=dev()),
                  garg_min=torch.empty((Q, Cout), dtype=torch.int32, device=dev()), group=group)
    Wd = cu(np.ascontiguousarray(W.T)) if transposed else cu(W)
    addkw = dict(add_group=add_group) if add_group else dict(add_index=cu(add_idx))
    ops.layer_fwd(cu(X), Wd, cu(b), P, Cin, Cout, in_scale=cu(scale), in_shift=cu(shift), in_relu=True,
                  addend=cu(addend), Y=Y, stat_partial=part, precision=1, w_transposed=transposed,
                  debug_flags=8 if single else 0, **addkw, **kw)
    torch.cuda.synchronize()
    if single:
        # plain TF32: both operands rounded to TF32, products accumulated in fp32
        A = np.maximum(X.astype(np.float64) * scale + shift, 0).astype(np.float32)
        ref = _layer_ref(_tf32(A), _tf32(W), b, None, None, False, addend, add_idx)
    else:
        ref = _layer_ref(X, W, b, scale, shift, True, addend, add_idx)
    Yh = Y.cpu().numpy()
    e = rel_err(Yh, ref)
    assert e < 2e-5, e
    ph = part.cpu().numpy()
    assert not np.isnan(ph).any(), "unwritten statistic slot"
    st = ph.astype(np.float64).sum(0)
    assert rel_err(st[0], ref.sum(0)) < 1e-4 and rel_err(st[1], (ref ** 2).sum(0)) < 1e-4
    if want_grp:
        Yg = Yh.reshape(P // group, group, Cout)
        assert np.array_equal(kw["gmax"].cpu().numpy(), Yg.max(1)) and np.array_equal(kw["gmin"].cpu().numpy(), Yg.min(1))
        assert np.array_equal(kw["garg_max"].cpu().numpy(), Yg.argmax(1))
        assert np.array_equal(kw["garg_min"].cpu().numpy(), Yg.argmin(1))


# The column tile is 128 wide when Cout % 128 == 0 and ceil(P / 128) * Cout / 128 >= the SM count (132 on an H100 SXM),
# else 64; the weight ring holds 4 K chunks at width 128 and 8 at width 64.
@pytest.mark.parametrize("P,Cin,Cout,group", [
    (5000, 32, 64, 0),            # one K chunk
    (4113, 64, 64, 0),            # panel resident (KC < ring), tail of 17 rows in the last 64-row tile
    (3000, 320, 64, 0),           # width 64, KC = 10 > 8 stages: the ring recycles
    (16996, 256, 256, 0),         # width 128, KC = 8 > 4 stages, tail of 100 rows in the last 128-row tile
    (17000, 256, 128, 0),         # 266 64-row tiles over 132 CTAs: CTA 0 gets 3, its warpgroups 2 and 1
    (192, 64, 64, 0),             # 3 64-row tiles over 2 CTAs: one CTA's second warpgroup has no tile at all
    (17024, 512, 128, 64),        # group 64 inside a warpgroup tile, odd tile counts, ring of width 128
    (16896, 256, 128, 128),       # group 128 across both warpgroups, width 128
    (8192, 96, 64, 128),          # group 128, width 64, KC = 3
    (16512, 64, 256, 16),
    (4160, 160, 128, 32),         # KC = 5 (odd), 65 64-row tiles
])
def test_layer_tc_shapes(P, Cin, Cout, group):
    _run_case(P, Cin, Cout, group)


@pytest.mark.parametrize("P,Cin,Cout", [(4100, 64, 128), (17000, 256, 256)])
def test_layer_tc_transposed_pack(P, Cin, Cout):
    """The dgrad call: W stored [Cin, Cout] and packed transposed."""
    _run_case(P, Cin, Cout, transposed=True)


@pytest.mark.parametrize("P,Cin,Cout,group", [(4100, 64, 128, 0), (16896, 256, 256, 64), (8192, 96, 64, 128)])
def test_layer_tc_single_precision(P, Cin, Cout, group):
    _run_case(P, Cin, Cout, group, single=True)


def test_layer_tc_add_group_and_transposed_single():
    _run_case(6400, 128, 128, 32, add_group=64)
    _run_case(4096, 256, 64, transposed=True, single=True)
