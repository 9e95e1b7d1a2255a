"""-m gpu: the activation ring of the wgmma layer kernel (csrc/mlp_tc.cu).  X reaches each consumer warpgroup through its
own ring of 3 tensor-map TMA stages, so these shapes cover what that path adds: X as a column view of a wider matrix
(ldx > Cin, the AGG[:, :C1] pattern of the detector head), K panels that wrap the ring inside a tile, row tails that the
TMA fills with zeros past P at both column widths, a CTA whose second warpgroup has no tile, and the group-128 combine
with the 128-wide column tile, whose epilogue runs in two 64-column halves.  Same reference and tolerances as
test_gpu_layer_tc."""
import numpy as np
import pytest
import torch

from tests.test_gpu_layer_tc import _run_case
from tests.test_gpu_ops import _layer_ref
from tests.util_gpu import cu, dev, rel_err

pytestmark = pytest.mark.gpu


# The column tile is 128 wide when Cout % 128 == 0 and ceil(P / 128) * Cout / 128 >= the SM count (132 on an H100 SXM),
# else 64; the activation ring holds 3 K chunks per warpgroup.
@pytest.mark.parametrize("P,Cin,Cout,group", [
    (5000, 160, 64, 0),           # KC = 5: the ring wraps inside a tile, and stage / phase shift from tile to tile
    (17000, 128, 128, 0),         # width 128, KC = 4
    (3001, 96, 64, 0),            # width 64, tail of 57 rows past P in the last 64-row tile
    (16900, 96, 128, 0),          # width 128, tail of 4 rows
    (130, 64, 128, 0),            # 3 64-row tiles over 2 x 2 CTAs: a second warpgroup without a tile, a 2-row tile
    (16896, 64, 256, 128),        # group 128 at width 128 (two column tiles): split epilogue + cross-warpgroup combine
    (16896, 320, 128, 64),        # group 64 at width 128, KC = 10
])
def test_layer_tc_ring_shapes(P, Cin, Cout, group):
    _run_case(P, Cin, Cout, group)


@pytest.mark.parametrize("P,Cin,Cout,ldx,col0,group", [
    (8192, 128, 512, 640, 0, 0),      # the head's AGG[:, :C1] view
    (8192, 128, 512, 640, 512, 0),    # a view that starts inside the row
    (16896, 128, 128, 256, 32, 16),   # width 128 with group outputs
    (4113, 64, 64, 96, 0, 0),         # width 64, row tail
])
def test_layer_tc_strided_x(P, Cin, Cout, ldx, col0, group):
    """X = B[:, col0:col0 + Cin] of a [P, ldx] matrix; the columns outside the view must not reach the product."""
    from usip_b200 import ops
    rng = np.random.default_rng(P + Cin + ldx + col0)
    B = rng.normal(size=(P, ldx)).astype(np.float32)
    X = B[:, col0:col0 + Cin]
    W = (rng.normal(size=(Cout, Cin)) / np.sqrt(Cin)).astype(np.float32)
    b = rng.normal(size=Cout).astype(np.float32)
    scale = rng.normal(size=Cin).astype(np.float32); shift = rng.normal(size=Cin).astype(np.float32)
    Bd = cu(B)
    Y = torch.empty((P, Cout), device=dev())
    nt = ops.stat_slots(P, Cout, 1, group, bool(group))
    part = torch.full((nt, 2, Cout), float("nan"), device=dev())
    kw = {}
    if group:
        kw = dict(gmax=torch.empty((P // group, Cout), device=dev()), gmin=torch.empty((P // group, Cout), device=dev()),
                  group=group)
    ops.layer_fwd(Bd[:, col0:col0 + Cin], cu(W), cu(b), P, Cin, Cout, in_scale=cu(scale), in_shift=cu(shift),
                  in_relu=True, Y=Y, stat_partial=part, precision=1, **kw)
    torch.cuda.synchronize()
    ref = _layer_ref(np.ascontiguousarray(X), W, b, scale, shift, True, None, None)
    Yh = Y.cpu().numpy()
    assert rel_err(Yh, ref) < 2e-5
    st = part.cpu().numpy().astype(np.float64).sum(0)
    assert rel_err(st[0], ref.sum(0)) < 1e-4 and rel_err(st[1], (ref ** 2).sum(0)) < 1e-4
    if group:
        Yg = Yh.reshape(P // group, group, Cout)
        assert np.array_equal(kw["gmax"].cpu().numpy(), Yg.max(1)) and np.array_equal(kw["gmin"].cpu().numpy(), Yg.min(1))
