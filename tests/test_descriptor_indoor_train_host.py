"""CPU: the host side of training the indoor descriptor -- the float64 restatement of DescCGFLoss the GPU tests use
(tests/cgf_ref.py) against the reference's own DescCGFLoss output stored in tests/golden/descriptor_indoor_train.npz, the
argument checks of the CGF kernels, and ModelDescriptorIndoor's refusals on a CPU device."""
import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests import cgf_ref
from tests.util_gpu import golden


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t if dtype is None else t.to(dtype)


@pytest.mark.parametrize("tag", ["train", "test"])
def test_restatement_selections_equal_the_reference(tag):
    """The restatement's picks, recomputed from the stored draws and the reference's transformed anchor keypoints, are the
    indices the reference's DescCGFLoss gathered."""
    g = golden("descriptor_indoor_train.npz")
    B, N, M, S, K, D, seed = [int(v) for v in g["cfg"]]
    cgf_radius = float(g["radii"][1])
    d = cgf_ref.train_inputs(B, N, M, S, seed, radius=cgf_radius)
    kt = cgf_ref.transform(_t(d["anc_kp"]), _t(d["R"]), _t(d["scale"]), _t(d["shift"]))
    assert torch.equal(kt, _t(g[tag + "/anc_kp_t"])), "the inputs no longer reproduce the golden's"
    near, far, out, mask = cgf_ref.selections(kt, _t(d["pos_kp"]), _t(g[tag + "/u_near"]), _t(g[tag + "/u_out"]), cgf_radius)
    for name, v in (("near", near), ("far", far), ("out", out)):
        assert np.array_equal(v.numpy(), g["%s/%s" % (tag, name)]), name
    share = float(mask.double().mean())
    assert 0.3 < share < 0.7, share                       # about half the anchors have a positive
    assert not mask.all(dim=1).any() and mask.any(dim=1).all()


def test_restatement_loss_equals_the_reference():
    """cgf_loss in float64 at the reference's picks, on the reference's descriptors, against the reference's DescCGFLoss
    output (float32 on the CPU) -- and its mean against the step's loss."""
    g = golden("descriptor_indoor_train.npz")
    B, N, M, S, K, D, seed = [int(v) for v in g["cfg"]]
    _, cgf_radius, gamma, smax = [float(v) for v in g["radii"]]
    d = cgf_ref.train_inputs(B, N, M, S, seed, radius=cgf_radius)
    kt = _t(g["train/anc_kp_t"])
    near, far, out, mask = cgf_ref.selections(kt, _t(d["pos_kp"]), _t(g["train/u_near"]), _t(g["train/u_out"]), cgf_radius)
    loss, active = cgf_ref.cgf_loss(_t(g["anc_desc"], torch.float64), _t(g["pos_desc"], torch.float64),
                                    _t(d["anc_sigma"], torch.float64), near, far, out, mask, _t(g["train/u_sel"]), gamma,
                                    smax)
    want = g["train/loss_vec"].astype(np.float64)
    assert np.abs(loss.numpy() - want).max() <= 1e-5 * np.abs(want).max()
    assert np.array_equal(active.numpy().astype(np.float32), g["train/active_vec"])
    assert abs(float(loss.mean()) - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))


def test_restatement_nan_cloud_and_fallbacks():
    """Every sigma >= sigma_max gives NaN weights, as the reference; an anchor with every positive inside the radius picks
    out = 0, one without a positive picks near = 0; duplicated positives tie `far` to the first index."""
    kp_p = torch.tensor([[[0.0, 0.0, -0.01, 0.0], [0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0]]])
    kp_a = torch.tensor([[[0.0, 5.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0]]])
    u = torch.rand((1, 4, 4), generator=torch.Generator().manual_seed(0))
    near, far, out, mask = cgf_ref.selections(kp_a, kp_p, u, u, 0.075)
    assert bool(mask[0, 0]) and int(out[0, 0]) == 0          # every positive inside: out falls back to index 0
    assert not bool(mask[0, 1]) and int(near[0, 1]) == 0
    assert int(far[0, 1]) == 0                               # positives 0, 1 and 3 coincide: the first index
    desc = torch.nn.functional.normalize(torch.randn((1, 8, 4), dtype=torch.float64), dim=1)
    loss, _ = cgf_ref.cgf_loss(desc, desc.flip(2), torch.full((1, 4), 0.6, dtype=torch.float64), near, far, out, mask,
                               torch.rand((1, 4)), 0.3, 0.5)
    assert bool(torch.isnan(loss).all())


def test_argument_checks_without_a_device():
    from usip_b200 import ops
    B, M, D = 2, 64, 64
    z = lambda *s: torch.zeros(s)
    args = lambda D=D, M=M: (z(B, 3, M), z(B, 3, M), z(B, D, M), z(B, D, M), z(B, M), (z(B, M, M), z(B, M, M), z(B, M)))
    assert ops.desc_cgf_check(*args()) == (B, M, D)
    with pytest.raises(ValueError, match="multiple of 4"):
        ops.desc_cgf_check(*args(D=66))
    with pytest.raises(ValueError, match="multiple of 4"):
        ops.desc_cgf_check(*args(D=ops.CGF_MAX_D + 4))
    with pytest.raises(ValueError, match="shared memory"):
        ops.desc_cgf_check(*args(M=ops.CGF_MAX_M + 1))
    a = list(args())
    a[2] = z(B, M, D).transpose(1, 2)
    with pytest.raises(ValueError, match="contiguous"):
        ops.desc_cgf_check(*a)
    a = list(args())
    a[4] = z(B, M).double()
    with pytest.raises(ValueError, match="float32"):
        ops.desc_cgf_check(*a)
    a = list(args())
    a[5] = (z(B, M, M), z(B, M, M), z(B, M - 1))
    with pytest.raises(ValueError, match="u_sel"):
        ops.desc_cgf_check(*a)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.desc_cgf(*args(), 0.075, 0.3, 0.5)             # valid shapes, but there is no CPU path


def _cpu_model():
    from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
    opt = ref_shim.make_opt(gpu_ids=[0], device=torch.device("cpu"), batch_size=1, input_pc_num=64, node_num=8,
                            ball_radius=0.75, ball_nsamples=448, descriptor_len=64, surface_normal_len=4,
                            CGF_radius=0.075, triple_loss_gamma=0.3, sigma_max=0.5)
    return ModelDescriptorIndoor(opt)


def test_cpu_device_refusals():
    from usip_b200.models import losses
    md = _cpu_model()
    assert md.optimizer_descriptor is None and isinstance(md.triplet_criteria, losses.DescCGFLoss)
    for call in (lambda: md.optimize(epoch=0), md.test_model):
        with pytest.raises(NotImplementedError, match="runs on CUDA tensors only; there is no CPU path"):
            call()
    with pytest.raises(NotImplementedError, match="DescCGFLoss"):
        md.triplet_criteria(z3 := torch.zeros(1, 3, 8), torch.zeros(1, 64, 8), z3, torch.zeros(1, 64, 8), torch.zeros(1, 8))
    with pytest.raises(NotImplementedError):
        md.get_current_visuals()
