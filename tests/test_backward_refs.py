"""The float64 reference formulas of tests/backward_ref.py (used by tests/test_gpu_backward_ops.py to check the backward
kernels) against torch.autograd of the forward they differentiate, in float64 on the CPU at small shapes."""
import torch

from tests import backward_ref as R

f64 = torch.float64


def _close(a, b, tol=1e-10):
    a, b = torch.as_tensor(a, dtype=f64), torch.as_tensor(b, dtype=f64)
    scale = max(float(b.abs().max()), 1e-30) if b.numel() else 1.0
    assert float((a - b).abs().max()) <= tol * scale, (float((a - b).abs().max()), scale)


def _bn_stats(y, eps=1e-5):
    mean = y.mean(0)
    invstd = 1.0 / torch.sqrt(y.var(0, unbiased=False) + eps)
    return mean, invstd


def test_bn_relu_bwd_ref_matches_autograd():
    g = torch.Generator().manual_seed(0)
    P, C = 37, 12
    for relu in (True, False):
        y = torch.randn(P, C, generator=g, dtype=f64).requires_grad_(True)
        gamma = torch.randn(C, generator=g, dtype=f64).requires_grad_(True)
        beta = torch.randn(C, generator=g, dtype=f64).requires_grad_(True)
        G = torch.randn(P, C, generator=g, dtype=f64)
        mean, invstd = _bn_stats(y)
        z = (y - mean) * invstd * gamma + beta
        out = z.clamp_min(0) if relu else z
        (out * G).sum().backward()
        m, i = mean.detach(), invstd.detach()
        scale = gamma.detach() * i
        shift = beta.detach() - m * scale
        gy, gg, gb = R.bn_relu_bwd(G, y.detach(), scale, shift, m, i, relu)
        _close(gy, y.grad); _close(gg, gamma.grad); _close(gb, beta.grad)


def test_groupmax_bwd_ref_matches_autograd():
    """out = max_k relu(bn(y)) with a unique maximum per (q, c); negative-scale channels select the group minimum of y."""
    g = torch.Generator().manual_seed(1)
    Q, K, C = 9, 16, 10
    y = torch.randn(Q * K, C, generator=g, dtype=f64).requires_grad_(True)
    gamma = torch.randn(C, generator=g, dtype=f64)
    gamma[::3] = -gamma[::3].abs()
    gamma = gamma.requires_grad_(True)
    beta = (torch.rand(C, generator=g, dtype=f64) + 0.5).requires_grad_(True)
    Gout = torch.randn(Q, C, generator=g, dtype=f64)
    mean, invstd = _bn_stats(y)
    z = ((y - mean) * invstd * gamma + beta).clamp_min(0).view(Q, K, C)
    z.max(1).values.mul(Gout).sum().backward()
    m, i = mean.detach(), invstd.detach()
    scale = gamma.detach() * i
    shift = beta.detach() - m * scale
    yv = y.detach().view(Q, K, C)
    gy, gg, gb, gz, argsel = R.groupmax_bwd(Gout, y.detach(), yv.argmax(1), yv.argmin(1), scale, m, i, shift)
    _close(gy, y.grad); _close(gg, gamma.grad); _close(gb, beta.grad)


def test_wgrad_ref_matches_autograd():
    g = torch.Generator().manual_seed(2)
    P, Cin, Cout = 50, 7, 5
    X = torch.randn(P, Cin, generator=g, dtype=f64)
    GY = torch.randn(P, Cout, generator=g, dtype=f64)
    sc, sh = torch.randn(Cin, generator=g, dtype=f64), torch.randn(Cin, generator=g, dtype=f64)
    for scale, shift, relu in ((sc, sh, True), (None, None, False), (None, None, True), (sc, sh, False)):
        W = torch.randn(Cout, Cin, generator=g, dtype=f64).requires_grad_(True)
        A = X if scale is None else X * scale + shift
        A = A.clamp_min(0) if relu else A
        (A @ W.t() * GY).sum().backward()
        _close(R.wgrad(GY, X, scale, shift, relu), W.grad)


def test_knn_combine_ref_matches_autograd():
    g = torch.Generator().manual_seed(3)
    B, M, K, C = 2, 11, 4, 6
    pts = torch.randn(B, 3, M, generator=g, dtype=f64)
    knn = torch.randint(0, M, (B, M, K), generator=g, dtype=torch.int32)
    knn[0, :, 0] = 3                                                   # a neighbour shared by every node
    Z = torch.randn(B * M, C, generator=g, dtype=f64).requires_grad_(True)
    W3 = torch.randn(C, 3, generator=g, dtype=f64).requires_grad_(True)
    bias = torch.randn(C, generator=g, dtype=f64)
    GY = torch.randn(B * M * K, C, generator=g, dtype=f64)
    Y = R.knn_combine_fwd(Z, pts, knn, W3, bias)
    # the forward itself, row by row
    for r in (0, 5, B * M * K - 1):
        b, m, k = r // (M * K), (r // K) % M, r % K
        j = int(knn[b, m, k])
        exp = Z[b * M + j] + W3 @ (pts[b, :, j] - pts[b, :, m]) + bias
        _close(Y[r].detach(), exp.detach())
    (Y * GY).sum().backward()
    GZ, gW = R.knn_combine_bwd(GY, pts, knn, B * M)
    _close(GZ, Z.grad); _close(gW, W3.grad)


def test_head_ref_matches_autograd():
    B, M = 2, 5
    g = torch.Generator().manual_seed(4)
    out4 = torch.randn(B * M, 4, generator=g, dtype=f64) * 3
    out4[0, 3], out4[1, 3], out4[2, 3] = 25.0, -40.0, 20.0               # above / far below / at the threshold
    out4 = out4.requires_grad_(True)
    cmean = torch.randn(B, 3, M, generator=g, dtype=f64)
    kp, sig = R.head_fwd(out4, cmean, 0.001)
    x = out4.detach()[:, 3]
    _close(sig.detach().view(-1), torch.nn.functional.softplus(x, beta=1, threshold=20) + 0.001)
    g_kp, g_sig = torch.randn(B, 3, M, generator=g, dtype=f64), torch.randn(B, M, generator=g, dtype=f64)
    ((kp * g_kp).sum() + (sig * g_sig).sum()).backward()
    _close(R.head_bwd(g_kp, g_sig, x, B, M), out4.grad)
    G0 = R.head_bwd(None, None, x, B, M)
    assert float(G0.abs().max()) == 0.0


def test_l2norm_ref_matches_autograd():
    g = torch.Generator().manual_seed(5)
    B, M, C = 2, 4, 7
    Y = torch.randn(B * M, C, generator=g, dtype=f64)
    Y[3] = 0.0                                                          # zero-norm row
    Y = Y.requires_grad_(True)
    out = R.l2norm_fwd(Y, B, M)
    gg = torch.randn(B, C, M, generator=g, dtype=f64)
    (out * gg).sum().backward()
    _close(R.l2norm_bwd(gg, Y.detach(), B, M), Y.grad)


def _triplet_case(seed):
    g = torch.Generator().manual_seed(seed)
    B, C, M, Mp, Mn = 2, 6, 9, 7, 5
    anc = torch.randn(B, C, M, generator=g, dtype=f64)
    pos = torch.randn(B, C, Mp, generator=g, dtype=f64)
    neg = torch.randn(B, C, Mn, generator=g, dtype=f64)
    ipos = torch.randint(0, Mp, (B, M), generator=g, dtype=torch.int32)
    ineg = torch.randint(0, Mn, (B, M), generator=g, dtype=torch.int32)
    ipos[:, :4] = 2                                                     # several anchors share one match
    pos[0, :, 3] = anc[0, :, 1]; ipos[0, 1] = 3                         # dpos = 0
    neg[1, :, 0] = anc[1, :, 2]; ineg[1, 2] = 0                         # dneg = 0
    sigma = torch.rand(B, M, generator=g, dtype=f64) * 2
    sigma[0, 5] = 3.5                                                   # sigma >= sigma_max: weight 0
    return anc, pos, neg, ipos, ineg, sigma


def test_desc_triplet_ref_matches_autograd():
    anc, pos, neg, ipos, ineg, sigma = _triplet_case(6)
    gamma, smax = 0.5, 3.0
    anc, pos, neg = (t.clone().requires_grad_(True) for t in (anc, pos, neg))
    dpos = (anc - R._col_gather(pos, ipos)).norm(dim=1)
    dneg = (anc - R._col_gather(neg, ineg)).norm(dim=1)
    loss, active = R.desc_triplet_fwd(dpos, dneg, sigma, gamma, smax)
    g_loss = torch.randn(loss.shape, generator=torch.Generator().manual_seed(7), dtype=f64)
    (loss * g_loss).sum().backward()
    ga, gp, gn = R.desc_triplet_bwd(anc.detach(), pos.detach(), neg.detach(), ipos, ineg, sigma, gamma, smax, g_loss)
    _close(ga, anc.grad); _close(gp, pos.grad); _close(gn, neg.grad)
    h = (dpos - dneg + gamma).detach()
    assert bool((h <= 0).any()) and bool((h > 0).any())                 # both hinge states occur


def test_transform_points_ref_matches_autograd():
    g = torch.Generator().manual_seed(8)
    B, M = 3, 6
    kp = torch.randn(B, 3, M, generator=g, dtype=f64).requires_grad_(True)
    Rm, sc, sh = torch.randn(B, 3, 3, generator=g, dtype=f64), torch.rand(B, generator=g, dtype=f64) + 0.5, torch.randn(B, 3, generator=g, dtype=f64)
    out = R.transform_points_fwd(kp, Rm, sc, sh)
    _close(out[1, :, 2].detach(), (Rm[1] @ kp[1, :, 2] * sc[1] + sh[1]).detach())
    go = torch.randn(B, 3, M, generator=g, dtype=f64)
    (out * go).sum().backward()
    _close(R.transform_points_bwd(go, Rm, sc), kp.grad)


def test_pairwise_min_bwd_ref_matches_autograd():
    g = torch.Generator().manual_seed(9)
    B, Ma, Nb = 2, 8, 5
    a = torch.randn(B, 3, Ma, generator=g, dtype=f64)
    b = torch.randn(B, 3, Nb, generator=g, dtype=f64)
    arg = torch.randint(0, Nb, (B, Ma), generator=g, dtype=torch.int32)
    arg[:, :3] = 1                                                      # repeated j
    a[0, :, 4] = b[0, :, int(arg[0, 4])]                                # d = 0
    for gv in (None, torch.randn(B, Ma, generator=g, dtype=f64)):
        aa, bb = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        d = (aa - R._col_gather(bb, arg)).norm(dim=1)
        (d * (1 if gv is None else gv) * 0.37).sum().backward()
        ga, gb = R.pairwise_min_bwd(a, b, d.detach(), arg, gv, 0.37)
        _close(ga, aa.grad); _close(gb, bb.grad)


def test_chamfer_prob_ref_matches_autograd():
    g = torch.Generator().manual_seed(10)
    B, M, N = 2, 7, 9
    src = torch.randn(B, 3, M, generator=g, dtype=f64)
    dst = torch.randn(B, 3, N, generator=g, dtype=f64)
    i_sd = torch.randint(0, N, (B, M), generator=g, dtype=torch.int32)
    i_ds = torch.randint(0, M, (B, N), generator=g, dtype=torch.int32)
    src[1, :, 2] = dst[1, :, int(i_sd[1, 2])]                           # d = 0
    ss, sd = torch.rand(B, M, generator=g, dtype=f64) + 0.2, torch.rand(B, N, generator=g, dtype=f64) + 0.2
    leaves = [t.clone().requires_grad_(True) for t in (src, dst, ss, sd)]
    loss, _, _ = R.chamfer_prob_fwd(*leaves, i_sd, i_ds)
    (loss * 1.7).backward()
    got = R.chamfer_prob_bwd(src, dst, ss, sd, i_sd, i_ds, 1.7)
    for a, leaf in zip(got, leaves):
        _close(a, leaf.grad)


def test_point_on_surface_ref_matches_autograd():
    g = torch.Generator().manual_seed(11)
    B, M, N, S = 2, 6, 10, 4
    kp = torch.randn(B, 3, M, generator=g, dtype=f64)
    pc = torch.randn(B, 3, N, generator=g, dtype=f64)
    sn = torch.randn(B, S, N, generator=g, dtype=f64)
    arg = torch.randint(0, N, (B, M), generator=g, dtype=torch.int32)
    kp[0, :, 1] = pc[0, :, int(arg[0, 1])]                              # r = 0
    kpl = kp.clone().requires_grad_(True)
    p, n = R._col_gather(pc, arg), R._col_gather(sn[:, :3], arg)
    d = kpl - p
    loss = ((n * d).sum(1) / (d.norm(dim=1) + 1e-7)) ** 2
    gv = torch.randn(B, M, generator=g, dtype=f64)
    (loss * gv).sum().backward()
    l_ref, g_ref = R.point_on_surface(kp, pc, sn, arg, gv)
    _close(l_ref, loss.detach()); _close(g_ref, kpl.grad)


def test_adam_reference_is_the_textbook_update():
    """adam_reference (torch.optim.Adam in float64) against the update written out, with an lr change and grad_scale."""
    g = torch.Generator().manual_seed(12)
    p0 = torch.randn(13, generator=g, dtype=f64)
    grads = [[torch.randn(13, generator=g, dtype=f64)] for _ in range(4)]
    lrs, (b1, b2), eps, gs = [1e-3, 1e-3, 5e-4, 5e-4], (0.9, 0.999), 1e-8, 0.5
    (p,), (m,), (v,) = R.adam_reference([p0], grads, lrs, (b1, b2), eps, gs)
    pe, me, ve = p0.clone(), torch.zeros(13, dtype=f64), torch.zeros(13, dtype=f64)
    for t, (gr, lr) in enumerate(zip(grads, lrs), 1):
        x = gr[0] * gs
        me = b1 * me + (1 - b1) * x
        ve = b2 * ve + (1 - b2) * x * x
        pe = pe - lr / (1 - b1 ** t) * me / (ve.sqrt() / (1 - b2 ** t) ** 0.5 + eps)
    _close(p, pe); _close(m, me); _close(v, ve)
