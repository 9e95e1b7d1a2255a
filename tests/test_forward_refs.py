"""The float64 reference formulas of tests/forward_ref.py (used by tests/test_gpu_forward_ops.py to check the forward
kernels) against the plain torch expressions of the reference they restate, in float64 on the CPU at small shapes."""
import torch
import torch.nn.functional as F

from tests import forward_ref as R

f64 = torch.float64


def _close(a, b, tol=1e-12):
    a, b = torch.as_tensor(a, dtype=f64), torch.as_tensor(b, dtype=f64)
    scale = max(float(b.abs().max()), 1e-30) if b.numel() else 1.0
    assert float((a - b).abs().max()) <= tol * scale, (float((a - b).abs().max()), scale)


def _index_max_loop(data, index, K):
    """index_max_cuda.cu:29-61 as written: one serial scan per (b, c), best starts at -1000 and index 0, '>' updates."""
    B, C, N = data.shape
    out = torch.zeros((B, C, K), dtype=torch.int64)
    for b in range(B):
        for c in range(C):
            best = [-1000.0] * K
            for n in range(N):
                k, v = int(index[b, n]), float(data[b, c, n])
                if v > best[k]:
                    best[k] = v
                    out[b, c, k] = n
    return out


def test_layer_fwd_ref_matches_conv1d():
    """MyConv2d (a 1x1 convolution) on the BatchNorm + ReLU output of the previous layer, plus a per-group addend."""
    g = torch.Generator().manual_seed(0)
    Pn, Cin, Cout, G = 40, 7, 5, 6
    X = torch.randn(Pn, Cin, generator=g, dtype=f64)
    W, b = torch.randn(Cout, Cin, generator=g, dtype=f64), torch.randn(Cout, generator=g, dtype=f64)
    sc, sh = torch.randn(Cin, generator=g, dtype=f64), torch.randn(Cin, generator=g, dtype=f64)
    add, ai = torch.randn(G, Cout, generator=g, dtype=f64), torch.randint(0, G, (Pn,), generator=g)
    a = torch.relu(X * sc + sh)
    ref = F.conv1d(a.t().unsqueeze(0), W.unsqueeze(2), b)[0].t() + add[ai]
    _close(R.layer_fwd(X, W, b, sc, sh, True, add, ai), ref)
    _close(R.layer_fwd(X, W), F.conv1d(X.t().unsqueeze(0), W.unsqueeze(2))[0].t())


def test_bn_train_and_eval_ref_match_batch_norm():
    g = torch.Generator().manual_seed(1)
    Pn, C = 37, 6
    Y = torch.randn(Pn, C, generator=g, dtype=f64) * 3 + torch.arange(C, dtype=f64)
    gamma, beta = torch.randn(C, generator=g, dtype=f64), torch.randn(C, generator=g, dtype=f64)
    rm, rv = torch.randn(C, generator=g, dtype=f64), torch.rand(C, generator=g, dtype=f64) + 0.5
    rm_t, rv_t = rm.clone(), rv.clone()
    ref = F.batch_norm(Y, rm_t, rv_t, gamma, beta, True, 0.1, 1e-5)
    scale, shift, mean, invstd, rm2, rv2 = R.bn_train(Y, gamma=gamma, beta=beta, eps=1e-5, momentum=0.1,
                                                       running_mean=rm, running_var=rv)
    _close(Y * scale + shift, ref)
    _close(rm2, rm_t); _close(rv2, rv_t)
    _close(mean, Y.mean(0)); _close(invstd, 1 / torch.sqrt(Y.var(0, unbiased=False) + 1e-5))
    s1, h1, *_ = R.bn_train(Y)                                                  # NULL gamma / beta: affine=False
    _close(Y * s1 + h1, F.batch_norm(Y, None, None, None, None, True, 0.1, 1e-5))
    es, eh = R.bn_eval(gamma, beta, rm, rv, 1e-5)
    _close(Y * es + eh, F.batch_norm(Y, rm, rv, gamma, beta, False, 0.1, 1e-5))


def test_group_select_ref_is_max_of_relu_bn():
    """The group max / min shortcut equals max_k relu(bn(y_k)) for negative, zero and positive scales."""
    g = torch.Generator().manual_seed(2)
    Q, K, C = 9, 8, 6
    Yg = torch.randn(Q, K, C, generator=g, dtype=f64)
    scale = torch.tensor([1.3, -0.7, 0.0, -0.0, 2.0, -2.5], dtype=f64)
    shift = torch.randn(C, generator=g, dtype=f64)
    ref = torch.stack([torch.relu(Yg[:, k] * scale + shift) for k in range(K)], 1).max(1).values
    _close(R.group_max_relu_bn(Yg, scale, shift), ref)
    _close(R.group_select(Yg.amax(1), Yg.amin(1), scale, shift), ref)


def test_softplus_ref_matches_torch_softplus():
    x = torch.tensor([-100.0, -30.0, -1.0, 0.0, 5.0, 19.5, 20.0, float(torch.nextafter(torch.tensor(20.0), torch.tensor(30.0))),
                      25.0], dtype=f64)
    assert torch.equal(R.softplus(x), torch.nn.Softplus()(x))
    x32 = torch.tensor([20.0, float(torch.nextafter(torch.tensor(20.0), torch.tensor(30.0)))], dtype=torch.float32)
    assert torch.equal(R.softplus(x32.double()).float(), torch.nn.Softplus()(x32))


def test_index_max_ref_matches_serial_scan():
    """Ties (first n), values at and below the floor, NaN, -0.0, empty clusters."""
    g = torch.Generator().manual_seed(3)
    B, C, N, K = 2, 5, 60, 9
    data = torch.round(torch.randn(B, C, N, generator=g, dtype=f64) * 2) / 2
    data[:, 1] = -2000.0
    data[:, 2, ::3] = -1000.0
    data[:, 3, ::4] = float("nan")
    data[:, 4, ::2] = -0.0
    index = torch.randint(0, K - 2, (B, N), generator=g)                          # the last two clusters empty
    assert torch.equal(R.index_max(data, index, K), _index_max_loop(data, index, K))


def _sorted_nodes(node_of_point, M):
    perm = torch.sort(node_of_point, dim=1, stable=True).indices
    counts = torch.stack([torch.bincount(r, minlength=M) for r in node_of_point])
    seg = torch.cat([torch.zeros(counts.shape[0], 1, dtype=torch.int64), counts.cumsum(1)], 1)
    return seg, perm


def test_segmax_ref_matches_index_max_gather():
    """networks.py:117-120: index_max on the (B, C, N) features, gather, times the non-empty mask."""
    g = torch.Generator().manual_seed(4)
    B, N, M, C = 2, 50, 7, 4
    node = torch.randint(0, M - 1, (B, N), generator=g)                            # node M-1 empty
    feat = torch.randn(B, C, N, generator=g, dtype=f64)
    feat[:, 1][node == 2] = -1500.0                                                # nothing above the floor
    seg, perm = _sorted_nodes(node, M)
    X = feat.gather(2, perm.unsqueeze(1).expand(B, C, N)).permute(0, 2, 1).reshape(B * N, C)
    pooled, arg = R.segmax(X, seg, perm)
    idx = _index_max_loop(feat, node, M)
    mask = torch.stack([torch.bincount(r, minlength=M) for r in node]) > 0
    ref = torch.gather(feat, 2, idx) * mask.unsqueeze(1)
    _close(pooled.view(B, M, C).permute(0, 2, 1), ref)
    rows = arg.view(B, M, C).permute(0, 2, 1)
    for b in range(B):
        for m in range(M):
            for c in range(C):
                if mask[b, m]:
                    assert int(perm[b, int(rows[b, c, m]) - b * N]) == int(idx[b, c, m])
                else:
                    assert int(rows[b, c, m]) == -1


def test_cluster_mean_decenter_ref_matches_networks_py():
    """networks.py:87-108: one-hot mask, sum / (count + 1e-5), x - mean of its node, cat sn."""
    g = torch.Generator().manual_seed(5)
    B, N, M, S = 2, 40, 6, 3
    x, sn = torch.randn(B, 3, N, generator=g, dtype=f64), torch.randn(B, S, N, generator=g, dtype=f64)
    node = torch.randint(0, M - 1, (B, N), generator=g)
    mask = F.one_hot(node, M).to(f64)                                              # (B, N, M)
    cm = (x.unsqueeze(3) * mask.unsqueeze(1)).sum(2) / (mask.sum(1).unsqueeze(1) + 1e-5)
    dec = x - torch.gather(cm, 2, node.unsqueeze(1).expand(B, 3, N))
    x_aug = torch.cat([dec, sn], 1)
    seg, perm = _sorted_nodes(node, M)
    cmean, rows = R.cluster_mean_decenter(x, sn, seg, perm)
    _close(cmean, cm)
    _close(rows.view(B, N, 3 + S), x_aug.gather(2, perm.unsqueeze(1).expand(B, 3 + S, N)).permute(0, 2, 1))


def test_knn_nodes_gather_and_pairmin_refs_match_torch():
    """torch.norm + topk(largest=False) (layers.py:417-421), the expand + gather of operations.py:271-287, and
    torch.norm + torch.min of DescPairScanLoss, with a duplicated point for the tie rule."""
    g = torch.Generator().manual_seed(6)
    B, M, K = 2, 12, 5
    pts = torch.randn(B, 3, M, generator=g, dtype=f64)
    d = torch.norm(pts.unsqueeze(3) - pts.unsqueeze(2), dim=1)
    assert torch.equal(R.knn_nodes(pts, K), d.topk(K, dim=2, largest=False, sorted=True).indices)
    pts[1, :, 9] = pts[1, :, 4]                                                    # exact tie: 4 before 9
    kn = R.knn_nodes(pts, M + 3)
    assert kn[1, 4, :2].tolist() == [4, 9] and kn[1, 9, :2].tolist() == [4, 9]
    assert bool((kn[:, :, M:] == 0).all())
    src = torch.randn(B, 4, M, generator=g, dtype=f64)
    idx = torch.randint(0, M, (B, M, K), generator=g)
    ref = torch.gather(src.unsqueeze(3).expand(B, 4, M, K), 2, idx.unsqueeze(1).expand(B, 4, M, K))
    assert torch.equal(R.knn_gather(src, idx), ref)
    a, b = torch.randn(B, 8, 10, generator=g, dtype=f64), torch.randn(B, 8, 15, generator=g, dtype=f64)
    b[0, :, 11] = b[0, :, 3]
    a[0, :, 2] = b[0, :, 3] + 1e-3
    mn, arg = R.desc_pairmin(a, b)
    dd = torch.norm(a.unsqueeze(3) - b.unsqueeze(2), dim=1)
    ref_v, ref_i = torch.min(dd, dim=2)
    _close(mn, ref_v)
    assert torch.equal(arg, ref_i) and int(arg[0, 2]) == 3


def test_chamfer_prob_terms_match_losses_py():
    """losses.py:79-97 with M != N: each direction's sigma pairs its own set with the nearest point of the other."""
    g = torch.Generator().manual_seed(7)
    B, M, N = 2, 9, 14
    src, dst = torch.randn(B, 3, M, generator=g, dtype=f64), torch.randn(B, 3, N, generator=g, dtype=f64)
    ss, sd = torch.rand(B, M, generator=g, dtype=f64) + 0.2, torch.rand(B, N, generator=g, dtype=f64) + 0.2
    D = torch.norm(src.unsqueeze(3) - dst.unsqueeze(2), dim=1)                     # (B, M, N)
    d_sd, i_sd = torch.min(D, dim=2)
    d_ds, i_ds = torch.min(D, dim=1)
    s1 = (ss + torch.gather(sd, 1, i_sd)) / 2
    s2 = (sd + torch.gather(ss, 1, i_ds)) / 2
    loss = torch.mean(torch.log(s1) + d_sd / s1) + torch.mean(torch.log(s2) + d_ds / s2)
    pure = torch.mean(d_sd) + torch.mean(d_ds)
    w1, w2 = (1 / s1) / torch.mean(1 / s1), (1 / s2) / torch.mean(1 / s2)
    weighted = torch.mean(d_sd * w1) + torch.mean(d_ds * w2)
    _close(R.chamfer_prob_terms(d_sd, i_sd, d_ds, i_ds, ss, sd), torch.stack([loss, pure, weighted]))
    _close(R.chamfer_prob_terms(d_sd, i_sd, d_ds, i_ds, ss, sd), torch.stack(list(R.chamfer_prob_fwd(src, dst, ss, sd, i_sd, i_ds))))
