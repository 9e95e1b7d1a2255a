"""The handcrafted keypoint baselines of evaluation/save_keypoints.py (methods 'iss', 'harris' and 'random',
:44-63 and :289-331), on the GPU, as drop-in detectors for the repeatability and registration evaluators.

    det = IssDetector()                          # save_keypoints.py:44-50 defaults
    res = KittiRepeatability(...).run(det)
    print(det.count_summary())                   # keypoint number max / min / mean, as save_keypoints.py:399-401

Each detector's run_model(pc, sn, node) returns (keypoints (B, 3, M), ranks (B, M)) like ModelDetector.run_model, with
M = node.shape[2]: the keypoints already in selection order and ranks 0, 1, ..., M - 1, so the evaluators' stable sort
by "sigma" keeps that order.  The order is ensure_keypoint_number for every K at once (usip_hc_select): the detected
keypoints in a Philox order, then the cloud's rows in a second Philox order, so that any K-prefix is K random keypoints
or every keypoint plus K - count random rows of the cloud.  `detected` holds each scan's keypoint count before that
padding, on the device: when it is far below K, the K-prefix is mostly random rows.

The random draws are keyed by (seed, batch number in the pass, cloud in the batch); Repeatability.detect calls
begin_pass() first, so two passes with one detector give identical results.

The kernels follow PCL's ISSKeypoint3D (without border estimation) and HarrisKeypoint3D (HARRIS response, normals over
the same radius, no refinement) as include/usip_b200.h states them.  Parity with PCL's own output, and with the
settings of the reference's PCLKeypoint module, is not established.
"""
import math

import torch

from usip_b200 import ops

METHODS = ("tsf", "iss", "harris", "random")


def _radius(name, r):
    r = float(r)
    if not (r > 0 and math.isfinite(r)):
        raise ValueError("%s must be finite and > 0, got %r" % (name, r))
    return r


class HandcraftedDetector:
    """Base of the three baselines: the selection, the step counter and the detected counts."""

    handcrafted = True
    method = None

    def __init__(self, seed=0):
        self.seed = int(seed)
        self.begin_pass()

    def begin_pass(self):
        """Restart the random stream: the next run_model call is batch 0 of a pass."""
        self.step = 0
        self._counts = []

    @property
    def detected(self):
        """Keypoints found per scan of the current pass before padding, (S,) i32 on the device."""
        if not self._counts:
            return torch.zeros((0,), dtype=torch.int32)
        return torch.cat(self._counts)

    def count_summary(self):
        """save_keypoints.py:399-401's line for the detected counts."""
        c = self.detected.cpu().double()
        if c.numel() == 0:
            return "keypoint number: no scan detected yet"
        return "keypoint number max: %d, min: %d, mean: %d" % (int(c.max()), int(c.min()), round(float(c.mean())))

    def flags(self, pc):
        """(B, N) i32 keypoint flags of pc (B, 3, N) f32 CUDA, or None for the random method."""
        raise NotImplementedError

    def run_model(self, pc, sn, node):
        pc = pc.contiguous()
        if pc.dtype != torch.float32 or not pc.is_cuda or pc.dim() != 3 or pc.shape[1] != 3:
            raise ValueError("pc must be a (B, 3, N) float32 CUDA tensor")
        B, _, N = pc.shape
        M = int(node.shape[2])
        if M > N:
            raise ValueError("%s: %d keypoints asked of %d-point clouds" % (type(self).__name__, M, N))
        flag = self.flags(pc)
        order, count = ops.hc_select(flag, B, N, M, self.seed, self.step, device=pc.device)
        self.step += 1
        self._counts.append(count)
        kp = torch.gather(pc, 2, order.long()[:, None, :].expand(B, 3, M))
        ranks = torch.arange(M, dtype=torch.float32, device=pc.device).expand(B, M).contiguous()
        return kp, ranks


class IssDetector(HandcraftedDetector):
    """'iss' (save_keypoints.py:44-50, :289-301): PCL ISSKeypoint3D without border estimation."""

    method = "iss"

    def __init__(self, salient_radius=2, non_max_radius=2, gamma_21=0.975, gamma_32=0.975, min_neighbors=5, seed=0):
        self.salient_radius = _radius("salient_radius", salient_radius)
        self.non_max_radius = _radius("non_max_radius", non_max_radius)
        for name, g in (("gamma_21", gamma_21), ("gamma_32", gamma_32)):
            if not 0 < float(g) <= 1:
                raise ValueError("%s must lie in (0, 1], got %r" % (name, g))
        self.gamma_21, self.gamma_32 = float(gamma_21), float(gamma_32)
        if int(min_neighbors) != min_neighbors or min_neighbors < 1:
            raise ValueError("min_neighbors must be an integer >= 1, got %r" % (min_neighbors,))
        self.min_neighbors = int(min_neighbors)
        super().__init__(seed)

    def flags(self, pc):
        grid = ops.hc_grid(pc)
        sal, _, _ = ops.iss_saliency(grid, self.salient_radius, self.gamma_21, self.gamma_32, self.min_neighbors)
        flag, _ = ops.hc_nonmax(grid, sal, self.non_max_radius, 0.0, True, self.min_neighbors)
        return flag


class Harris3DDetector(HandcraftedDetector):
    """'harris' (save_keypoints.py:52-55, :302-311): PCL HarrisKeypoint3D, HARRIS response, no refinement."""

    method = "harris"

    def __init__(self, radius=1, threshold=0.001, seed=0):
        self.radius = _radius("radius", radius)
        if not math.isfinite(float(threshold)):
            raise ValueError("threshold must be finite, got %r" % (threshold,))
        self.threshold = float(threshold)
        super().__init__(seed)

    def flags(self, pc):
        grid = ops.hc_grid(pc)
        resp, _, _ = ops.harris3d_response(grid, self.radius)
        flag, _ = ops.hc_nonmax(grid, resp, self.radius, self.threshold, False, 1)
        return flag


class RandomDetector(HandcraftedDetector):
    """'random' (save_keypoints.py:325-330): M rows of the cloud drawn without replacement."""

    method = "random"

    def flags(self, pc):
        return None


# ----------------------------------------------------------------------------------------------- command line
def add_method_args(ap):
    """--method and the baselines' parameters (save_keypoints.py:44-55 defaults)."""
    g = ap.add_argument_group("detector method")
    g.add_argument("--method", choices=METHODS, default="tsf",
                   help="tsf: the trained detector (the default); iss, harris, random: the handcrafted baselines")
    g.add_argument("--iss-salient-radius", type=float, default=2.0)
    g.add_argument("--iss-non-max-radius", type=float, default=2.0)
    g.add_argument("--iss-gamma-21", type=float, default=0.975)
    g.add_argument("--iss-gamma-32", type=float, default=0.975)
    g.add_argument("--iss-min-neighbors", type=int, default=5)
    g.add_argument("--harris-radius", type=float, default=1.0)
    g.add_argument("--harris-threshold", type=float, default=0.001)


def detector_from_args(a, ap):
    """The handcrafted detector --method names (None for tsf); bad parameters end the program through ap.error."""
    try:
        if a.method == "iss":
            return IssDetector(a.iss_salient_radius, a.iss_non_max_radius, a.iss_gamma_21, a.iss_gamma_32,
                               a.iss_min_neighbors, seed=a.seed)
        if a.method == "harris":
            return Harris3DDetector(a.harris_radius, a.harris_threshold, seed=a.seed)
        if a.method == "random":
            return RandomDetector(seed=a.seed)
    except ValueError as e:
        ap.error(str(e))
    return None
