"""Plain float64 restatements of the backward kernels of csrc/backward.cu, csrc/loss.cu and csrc/optim.cu.

Every function takes and returns torch float64 tensors on any device (the -m gpu tests run them on the GPU next to the
kernel under test, tests/test_backward_refs.py checks each one against torch.autograd on the CPU).  Discrete decisions
(arg-max rows, neighbour indices, ReLU masks) are inputs or are recomputed from the same float64 values, so a caller that
builds its data with margin gets the same decisions as the kernel."""
import torch


def bn_relu_bwd(G, Y, scale, shift, mean, invstd, relu):
    """Train-mode BatchNorm(+ReLU) backward from the saved statistics (the formula of usip_bn_bwd_*):
    g_z = G * 1[scale*y + shift > 0], xhat = (y - mean) * invstd,
    g_y = scale * (g_z - mean_r(g_z) - xhat * mean_r(g_z * xhat)); g_beta = sum_r g_z, g_gamma = sum_r g_z * xhat."""
    gz = G * ((Y * scale + shift) > 0) if relu else G
    xhat = (Y - mean) * invstd
    g_beta = gz.sum(0)
    g_gamma = (gz * xhat).sum(0)
    n = Y.shape[0]
    gy = scale * (gz - g_beta / n - xhat * (g_gamma / n))
    return gy, g_gamma, g_beta


def groupmax_bwd(Gout, Y, argmax, argmin, scale, mean, invstd, shift):
    """Backward of out[q,c] = max_k relu(scale*y[q*K+k,c] + shift) through train-mode BN, with the maximum at row
    (scale >= 0 ? argmax : argmin)[q,c] of group q.  Y [Q*K, C]; returns (g_y [Q*K,C], g_gamma, g_beta, gz [Q,C], argsel)."""
    Q, C = Gout.shape
    K = Y.shape[0] // Q
    argsel = torch.where(scale >= 0, argmax, argmin).long()
    ysel = Y.view(Q, K, C).gather(1, argsel.unsqueeze(1)).squeeze(1)
    gz = Gout * ((ysel * scale + shift) > 0)
    dense = torch.zeros((Q, K, C), dtype=Y.dtype, device=Y.device)
    dense.scatter_(1, argsel.unsqueeze(1), gz.unsqueeze(1))
    gy, g_gamma, g_beta = bn_relu_bwd(dense.view(Q * K, C), Y, scale, shift, mean, invstd, False)
    return gy, g_gamma, g_beta, gz, argsel


def wgrad(GY, X, in_scale=None, in_shift=None, in_relu=False):
    """gW[Cout, Cin] = GY^T act(X), act = optional affine then optional ReLU."""
    A = X if in_scale is None else X * in_scale + in_shift
    if in_relu:
        A = A.clamp_min(0)
    return GY.t() @ A


def knn_combine_fwd(Z, pts, knn_idx, W3, bias):
    """Y[(b,m,k), c] = Z[b*M + j, c] + sum_t W3[c,t] * (pts[b,t,j] - pts[b,t,m]) + bias[c], j = knn_idx[b,m,k]."""
    B, _, M = pts.shape
    K = knn_idx.shape[2]
    j = knn_idx.long()
    rows = (torch.arange(B, device=pts.device).view(B, 1, 1) * M + j).reshape(-1)
    delta = _knn_delta(pts, j)                                              # [B*M*K, 3]
    return Z[rows] + delta @ W3.t() + (0 if bias is None else bias)


def _knn_delta(pts, j):
    """pts[b,:,j] - pts[b,:,m] of every row (b,m,k) as [B*M*K, 3]."""
    B, _, M = pts.shape
    K = j.shape[2]
    pj = torch.gather(pts, 2, j.reshape(B, 1, M * K).expand(B, 3, M * K)).view(B, 3, M, K)
    d = pj - pts.unsqueeze(3)
    return d.permute(0, 2, 3, 1).reshape(B * M * K, 3)


def knn_combine_bwd(GY, pts, knn_idx, Q):
    """(G_Z [Q, C], gWxyz [C, 3]) of knn_combine_fwd: G_Z[b*M + j] += GY[row], gWxyz = GY^T delta."""
    B, _, M = pts.shape
    j = knn_idx.long()
    rows = (torch.arange(B, device=pts.device).view(B, 1, 1) * M + j).reshape(-1)
    GZ = torch.zeros((Q, GY.shape[1]), dtype=GY.dtype, device=GY.device).index_add_(0, rows, GY)
    return GZ, GY.t() @ _knn_delta(pts, j)


def head_fwd(out4, cmean, lb):
    """keypoints (B,3,M) = out4[:, 0:3] + cluster_mean; sigmas (B,M) = softplus(out4[:, 3]) (threshold 20) + lb."""
    B, _, M = cmean.shape
    o = out4.view(B, M, -1)
    kp = o[:, :, :3].permute(0, 2, 1) + cmean
    x = o[:, :, 3]
    sig = torch.where(x > 20, x, torch.log1p(torch.exp(torch.clamp(x, max=20)))) + lb
    return kp, sig


def head_bwd(g_kp, g_sig, x, B, M):
    """G [B*M, 4]: columns 0:3 = g_kp (B,3,M) as rows, column 3 = g_sig * sigmoid(x) (1 above 20)."""
    dev = x.device
    G = torch.zeros((B * M, 4), dtype=torch.float64, device=dev)
    if g_kp is not None:
        G[:, :3] = g_kp.permute(0, 2, 1).reshape(B * M, 3)
    if g_sig is not None:
        G[:, 3] = g_sig.reshape(-1) * torch.where(x > 20, torch.ones_like(x), torch.sigmoid(x))
    return G


def l2norm_fwd(Y, B, M):
    """(B, C, M) = Y[q] / (||Y[q]|| + 1e-5) of the [B*M, C] rows Y."""
    n = Y.norm(dim=1, keepdim=True)
    return (Y / (n + 1e-5)).view(B, M, -1).permute(0, 2, 1)


def l2norm_bwd(g, Y, B, M):
    """g (B,C,M) -> g_y [B*M, C] = g/(n+eps) - y (g.y) / (n (n+eps)^2); a zero row (n = 0) gets g/eps."""
    gr = g.permute(0, 2, 1).reshape(B * M, -1)
    n = Y.norm(dim=1, keepdim=True)
    d = n + 1e-5
    gy = (gr * Y).sum(1, keepdim=True)
    k = torch.where(n > 0, gy / (n * d * d).clamp_min(1e-300), torch.zeros_like(n))
    return gr / d - Y * k


def triplet_weights(sigma, sigma_max):
    w = (sigma_max - sigma).clamp_min(0)
    return w / w.mean(1, keepdim=True)


def desc_triplet_fwd(dpos, dneg, sigma, gamma, sigma_max):
    """loss (B,M) = w * clamp(dpos - dneg + gamma, 0), active (B) = mean(dpos - dneg + gamma > 0)."""
    h = dpos - dneg + gamma
    return triplet_weights(sigma, sigma_max) * h.clamp_min(0), (h > 0).double().mean(1)


def _col_gather(x, idx):
    """x (B,C,L), idx (B,M) -> (B,C,M)."""
    return torch.gather(x, 2, idx.long().unsqueeze(1).expand(-1, x.shape[1], -1))


def desc_triplet_bwd(anc, pos, neg, ipos, ineg, sigma, gamma, sigma_max, g_loss):
    """Gradients (g_anc, g_pos, g_neg) of sum g_loss * w * clamp(||a - pos[ipos]|| - ||a - neg[ineg]|| + gamma, 0),
    w detached; torch.norm's zero sub-gradient where a distance is 0."""
    dp_v = anc - _col_gather(pos, ipos)
    dn_v = anc - _col_gather(neg, ineg)
    dpos, dneg = dp_v.norm(dim=1), dn_v.norm(dim=1)
    coef = g_loss * triplet_weights(sigma, sigma_max) * ((dpos - dneg + gamma) > 0)
    ip = torch.where(dpos > 0, coef / dpos.clamp_min(1e-300), torch.zeros_like(dpos)).unsqueeze(1)
    inn = torch.where(dneg > 0, coef / dneg.clamp_min(1e-300), torch.zeros_like(dneg)).unsqueeze(1)
    tp, tn = dp_v * ip, dn_v * inn
    g_pos = torch.zeros_like(pos).scatter_add_(2, ipos.long().unsqueeze(1).expand_as(tp), -tp)
    g_neg = torch.zeros_like(neg).scatter_add_(2, ineg.long().unsqueeze(1).expand_as(tn), tn)
    return tp - tn, g_pos, g_neg


def transform_points_fwd(kp, R, scale, shift):
    return (R @ kp) * scale.view(-1, 1, 1) + shift.view(-1, 3, 1)


def transform_points_bwd(g, R, scale):
    return (R.transpose(1, 2) @ g) * scale.view(-1, 1, 1)


def pairwise_min_bwd(a, b, d, arg, g, gscale):
    """(grad_a, grad_b) of sum_i g_i * gscale * ||a_i - b_arg(i)||, zero where d == 0; g None means ones."""
    w = (torch.ones_like(d) if g is None else g) * gscale
    diff = a - _col_gather(b, arg)
    inv = torch.where(d > 0, w / d.clamp_min(1e-300), torch.zeros_like(d)).unsqueeze(1)
    ga = diff * inv
    gb = torch.zeros_like(b).scatter_add_(2, arg.long().unsqueeze(1).expand_as(ga), -ga)
    return ga, gb


def chamfer_prob_fwd(src, dst, sig_src, sig_dst, i_sd, i_ds):
    """ChamferLoss_Brute's sigma branch with the nearest neighbours given: (loss, chamfer_pure, chamfer_weighted)."""
    d_sd = (src - _col_gather(dst, i_sd)).norm(dim=1)
    d_ds = (dst - _col_gather(src, i_ds)).norm(dim=1)
    s_sd = 0.5 * (sig_src + torch.gather(sig_dst, 1, i_sd.long()))
    s_ds = 0.5 * (sig_dst + torch.gather(sig_src, 1, i_ds.long()))
    loss = (torch.log(s_sd) + d_sd / s_sd).mean() + (torch.log(s_ds) + d_ds / s_ds).mean()
    pure = d_sd.mean() + d_ds.mean()
    weighted = (d_sd / s_sd).mean() / (1 / s_sd).mean() + (d_ds / s_ds).mean() / (1 / s_ds).mean()
    return loss, pure, weighted


def chamfer_prob_bwd(src, dst, sig_src, sig_dst, i_sd, i_ds, gout):
    """(g_src, g_dst, g_sig_src, g_sig_dst) of gout * loss (chamfer_prob_fwd), zero distance sub-gradient 0."""
    g_src, g_dst = torch.zeros_like(src), torch.zeros_like(dst)
    g_ss, g_sd = torch.zeros_like(sig_src), torch.zeros_like(sig_dst)
    for A, Bm, sa, sb, idx, gA, gB, gsa, gsb in ((src, dst, sig_src, sig_dst, i_sd, g_src, g_dst, g_ss, g_sd),
                                                 (dst, src, sig_dst, sig_src, i_ds, g_dst, g_src, g_sd, g_ss)):
        n = A.shape[0] * A.shape[2]
        diff = A - _col_gather(Bm, idx)
        d = diff.norm(dim=1)
        s = 0.5 * (sa + torch.gather(sb, 1, idx.long()))
        w = gout / n
        gd = w / s
        gs = w * (1 / s - d / (s * s)) * 0.5
        gsa.add_(gs)
        gsb.scatter_add_(1, idx.long(), gs)
        v = diff * torch.where(d > 0, gd / d.clamp_min(1e-300), torch.zeros_like(d)).unsqueeze(1)
        gA.add_(v)
        gB.scatter_add_(2, idx.long().unsqueeze(1).expand_as(v), -v)
    return g_src, g_dst, g_ss, g_sd


def point_on_surface(kp, pc, sn, arg, g):
    """(loss (B,M), g_kp (B,3,M)): loss = (n . (kp - p) / (||kp - p|| + 1e-7))^2 at p = pc[:, arg], n = sn[0:3, arg];
    dloss/dkp = 2 s (n/e - d (n.d) / (r e^2)), the second term 0 at r = 0."""
    p = _col_gather(pc, arg)
    n = _col_gather(sn[:, :3], arg)
    d = kp - p
    r = d.norm(dim=1, keepdim=True)
    e = r + 1e-7
    s = (n * d).sum(1, keepdim=True) / e
    nd = (n * d).sum(1, keepdim=True)
    c = torch.where(r > 0, nd / (r * e * e).clamp_min(1e-300), torch.zeros_like(r))
    gk = None if g is None else 2 * s * g.unsqueeze(1) * (n / e - d * c)
    return (s * s).squeeze(1), gk


def adam_reference(params, grads_per_step, lrs, betas, eps, grad_scale):
    """torch.optim.Adam in float64 on copies of `params` (list of tensors); grads_per_step[t][i] is the raw gradient of
    parameter i at step t (multiplied by grad_scale before the update), lrs[t] the learning rate of step t."""
    ps = [p.detach().double().clone().requires_grad_(True) for p in params]
    opt = torch.optim.Adam(ps, lr=lrs[0], betas=betas, eps=eps, weight_decay=0, foreach=False)
    for gs, lr in zip(grads_per_step, lrs):
        for g_ in opt.param_groups:
            g_["lr"] = lr
        for p, g in zip(ps, gs):
            p.grad = g.double() * grad_scale
        opt.step()
    st = [opt.state[p] for p in ps]
    return [p.detach() for p in ps], [s["exp_avg"] for s in st], [s["exp_avg_sq"] for s in st]
