"""References for DescCGFLoss (models/losses.py:240-369), the indoor descriptor's triplet loss, and the inputs of its tests.

* selections: the reference's three picks per anchor, restated literally in torch on the given device and dtype: the
  keypoint distance sqrt((dx*dx + dy*dy) + dz*dz) (the kernel's fp32 order; torch.norm sums the same three squares),
  mask = d <= CGF_radius, near = argmax(mask * u_near), far = argmin(d + mask * 1000), out = argmax(!mask * u_out), first
  index on ties.
* cgf_loss: the loss and active share from pinned picks, differentiable in the descriptors (float64 for the gradient
  checks), term for term the reference's expression.
* train_inputs: an (anchor, positive) batch in the layout of ModelDescriptorIndoor.set_input, where about half the anchors
  have a positive keypoint within CGF_radius and no keypoint pair lies within MARGIN of that radius, so the fp32 rounding
  of the anchor transform cannot move a pick.
"""
import numpy as np
import torch

MARGIN = 1e-4


def keypoint_dist(anc_kp, pos_kp):
    """(B,3,M), (B,3,M) -> (B,M,M): d[b,m,j] = sqrt((dx*dx + dy*dy) + dz*dz), dx = anc[b,0,m] - pos[b,0,j]."""
    d = anc_kp[:, :, :, None] - pos_kp[:, :, None, :]
    return torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def selections(anc_kp, pos_kp, u_near, u_out, radius):
    """-> near, far, out (B,M) int64 and mask (B,M) bool (the anchor has a positive keypoint within radius)."""
    d = keypoint_dist(anc_kp, pos_kp)
    inside = d <= radius
    near = torch.max(inside.to(u_near.dtype) * u_near, dim=2)[1]
    far = torch.min(d + inside.to(d.dtype) * 1000, dim=2)[1]
    out = torch.max(u_out * (~inside).to(u_out.dtype), dim=2)[1]
    return near, far, out, inside.any(dim=2)


def _pair_dist(anc, pos, idx):
    """||anc[:, :, m] - pos[:, :, idx[b, m]]||_2 -> (B,M)."""
    p = torch.gather(pos, 2, idx.unsqueeze(1).expand(-1, pos.shape[1], -1))
    return torch.sqrt(((anc - p) ** 2).sum(1))


def cgf_loss(anc, pos, sigmas, near, far, out, mask, u_sel, gamma, sigma_max):
    """losses.py:283-326 at pinned picks: anc, pos (B,D,M) -> (loss (B,M), active (B))."""
    M = anc.shape[2]
    maskf = mask.to(anc.dtype)
    positive = _pair_dist(anc, pos, near)
    sel = (u_sel < 0.5).to(anc.dtype)
    negative = sel * _pair_dist(anc, pos, far) + (1 - sel) * _pair_dist(anc, pos, out)
    scaling = M / (maskf.sum(1) + 1)
    before = (positive - negative + gamma) * maskf
    active = (before > 1e-5).to(anc.dtype).sum(1) / (maskf.sum(1) + 1)
    w = torch.clamp(sigma_max - sigmas.to(anc.dtype), min=0)
    w = (w / w.mean(1, keepdim=True)).detach()
    return w * torch.clamp(before, min=0) * scaling.unsqueeze(1), active


def transform(kp, R, scale, shift):
    """keypoint_descriptor.py:474-477: R @ kp * scale + shift; R (B,3,3), scale (B,) (the loader's per-pair float),
    shift (B,3,1)."""
    return torch.matmul(R, kp) * scale.unsqueeze(1).unsqueeze(2) + shift


def _rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def train_inputs(B, N, M, S, seed, radius=0.075, half=1.0, share=0.5):
    """-> dict of float32 arrays: anc_pc/pos_pc (B,3,N), anc_sn/pos_sn (B,S,N), anc_kp/pos_kp (B,3,M), anc_sigma/pos_sigma
    (B,M), R (B,3,3), scale (B,), shift (B,3,1).  The anchor cloud is the positive cloud mapped back through (R, scale,
    shift) with a little noise; `share` of the anchors land within radius of a positive keypoint (in the positive frame),
    the others further away, and every pair distance stays MARGIN away from radius."""
    rng = np.random.default_rng(seed)
    pos_pc = rng.uniform(-half, half, (B, 3, N))
    sn = rng.normal(0, 1, (B, S, N)).astype(np.float32)
    pos_kp = np.take_along_axis(pos_pc, rng.integers(0, N, (B, 1, M)), 2) + rng.normal(0, 0.02, (B, 3, M))
    R = np.stack([_rotation(rng) for _ in range(B)])
    scale = rng.uniform(0.8, 1.2, B)
    shift = rng.uniform(-0.3, 0.3, (B, 3, 1))
    anc_t = np.empty((B, 3, M))
    for b in range(B):
        for m in range(M):
            for _ in range(1000):
                if rng.random() < share:             # near a positive keypoint, well inside the radius
                    v = rng.normal(size=3)
                    p = pos_kp[b, :, rng.integers(M)] + v / np.linalg.norm(v) * rng.uniform(0, 0.8 * radius)
                else:
                    p = pos_pc[b, :, rng.integers(N)] + rng.normal(0, 0.05, 3)
                d = np.linalg.norm(pos_kp[b] - p[:, None], axis=0)
                if np.abs(d - radius).min() >= 2 * MARGIN:
                    anc_t[b, :, m] = p
                    break
            else:
                raise RuntimeError("no anchor placement keeps the margin")
    inv = lambda x: np.einsum("bji,bjn->bin", R, (x - shift) / scale[:, None, None])   # R^T (x - shift) / scale
    anc_pc = inv(pos_pc) + rng.normal(0, 1e-3, (B, 3, N))
    out = dict(anc_pc=anc_pc, anc_sn=sn, anc_kp=inv(anc_t), anc_sigma=rng.uniform(0.05, 0.6, (B, M)),
               pos_pc=pos_pc, pos_sn=sn.copy(), pos_kp=pos_kp, pos_sigma=rng.uniform(0.05, 0.6, (B, M)),
               R=R, scale=scale, shift=shift)
    out = {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in out.items()}
    # the margin must survive the fp32 keypoints and transform
    kt = transform(torch.from_numpy(out["anc_kp"]), torch.from_numpy(out["R"]), torch.from_numpy(out["scale"]),
                   torch.from_numpy(out["shift"]))
    d = keypoint_dist(kt, torch.from_numpy(out["pos_kp"])).double()
    assert float((d - radius).abs().min()) >= MARGIN, float((d - radius).abs().min())
    return out


SET_INPUT_KEYS = ("anc_pc", "anc_sn", "anc_kp", "anc_sigma", "pos_pc", "pos_sn", "pos_kp", "pos_sigma", "R", "scale", "shift")
