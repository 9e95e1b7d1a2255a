"""Plain float64 restatements of the forward kernels of csrc/mlp.cu, csrc/group.cu and csrc/loss.cu.

Every function takes and returns torch tensors on any device (the -m gpu tests of tests/test_gpu_forward_ops.py run them
on the GPU next to the kernel under test; tests/test_forward_refs.py checks each one against the plain torch expression
of the reference on the CPU).  Discrete choices come out as indices: arg-max rows, nearest indices, neighbour lists.
The forward formulas that tests/backward_ref.py already states (knn_combine_fwd, head_fwd, l2norm_fwd,
desc_triplet_fwd, transform_points_fwd, chamfer_prob_fwd, point_on_surface) are re-exported here, not restated."""
import torch

from tests.backward_ref import (_col_gather, chamfer_prob_fwd, desc_triplet_fwd, head_fwd,  # noqa: F401
                                knn_combine_fwd, l2norm_fwd, point_on_surface, transform_points_fwd)

FLOOR = -1000.0          # index_max_cuda.cu:38: only values above it can win


def layer_fwd(X, W, bias=None, in_scale=None, in_shift=None, in_relu=False, addend=None, add_index=None):
    """usip_layer_fwd: Y = act(X) W^T + bias (+ addend[add_index]), act = folded BN affine then ReLU of the previous
    layer (layers.py:172-216 MyConv2d after MyBatchNorm + ReLU, :248-303).  X [P, Cin], W [Cout, Cin]."""
    A = X if in_scale is None else X * in_scale + in_shift
    if in_relu:
        A = A.clamp_min(0)
    Y = A @ W.t()
    if bias is not None:
        Y = Y + bias
    if addend is not None:
        Y = Y + addend[add_index.long()]
    return Y


def bn_train_from_sums(S, SS, count, gamma=None, beta=None, eps=1e-5, momentum=0.1, running_mean=None, running_var=None):
    """Train-mode F.batch_norm (layers.py:69-71) from per-channel sums S = sum y and SS = sum y^2 over `count` rows, as
    usip_bn_finalize folds it: mean = S/n, var = SS/n - mean^2 (biased, clamped at 0), invstd = 1/sqrt(var + eps),
    scale = gamma invstd, shift = beta - mean scale; running stats move by `momentum` toward mean and the unbiased var
    (the biased one when n == 1, where the unbiased one is undefined).  Returns
    (scale, shift, mean, invstd, new running_mean or None, new running_var or None)."""
    mean = S / count
    var = (SS / count - mean * mean).clamp_min(0)
    invstd = 1.0 / torch.sqrt(var + eps)
    g = torch.ones_like(S) if gamma is None else gamma
    b = torch.zeros_like(S) if beta is None else beta
    scale = g * invstd
    shift = b - mean * scale
    rm = rv = None
    if running_mean is not None:
        rm = (1 - momentum) * running_mean + momentum * mean
    if running_var is not None:
        unb = var * count / (count - 1) if count > 1 else var
        rv = (1 - momentum) * running_var + momentum * unb
    return scale, shift, mean, invstd, rm, rv


def bn_train(Y, **kw):
    """bn_train_from_sums over the rows of Y [P, C]."""
    return bn_train_from_sums(Y.sum(0), (Y * Y).sum(0), Y.shape[0], **kw)


def bn_eval(gamma, beta, running_mean, running_var, eps=1e-5):
    """Eval-mode F.batch_norm folded into (scale, shift) = (gamma / sqrt(rv + eps), beta - rm scale)."""
    scale = gamma / torch.sqrt(running_var + eps)
    return scale, beta - running_mean * scale


def group_max_relu_bn(Yg, scale, shift):
    """max_k relu(bn(y_k)) of layers.py:433,438: Yg (Q, K, C) raw outputs -> (Q, C)."""
    return (Yg * scale + shift).clamp_min(0).amax(1)


def group_select(gmax, gmin, scale, shift):
    """usip_group_select: the same value from the group max and min of the raw outputs alone (relu o affine is monotone:
    the max for scale >= 0, the min otherwise)."""
    return (torch.where(scale >= 0, gmax, gmin) * scale + shift).clamp_min(0)


def softplus(x):
    """torch.nn.Softplus() (beta 1, threshold 20) of networks.py:72: x itself above 20, log(1 + e^x) otherwise."""
    return torch.where(x > 20, x, torch.log1p(torch.exp(torch.clamp(x, max=20))))


def index_max(data, index, K):
    """index_max_cuda.cu:29-61: data (B, C, N), index (B, N) in [0, K) -> (B, C, K) int64, the smallest n attaining
    max{data[b, c, n] : index[b, n] == k, data > -1000} ('>' on every step: NaN never wins, -0 equals +0), else 0."""
    B, C, N = data.shape
    idx = index.long().unsqueeze(1).expand(B, C, N)
    vals = torch.where(data > FLOOR, data, torch.full_like(data, -float("inf")))
    best = torch.full((B, C, K), -float("inf"), dtype=data.dtype, device=data.device).scatter_reduce(
        2, idx, vals, "amax", include_self=True)
    hit = (vals == best.gather(2, idx)) & (vals > -float("inf"))
    n = torch.arange(N, device=data.device).expand(B, C, N)
    first = torch.full((B, C, K), N, dtype=torch.int64, device=data.device).scatter_reduce(
        2, idx, torch.where(hit, n, torch.full_like(n, N)), "amin", include_self=True)
    return torch.where(first == N, torch.zeros_like(first), first)


def segmax(X, seg_off, perm):
    """usip_segmax: index_max + gather * mask_row_max (networks.py:117-120,130-133) over the rows of X [B*N, C] sorted
    by node (rows seg_off[b, m] .. seg_off[b, m+1] of cloud b belong to node m, sorted row r is point perm[b, r]).
    -> pooled [B*M, C] (0 for an empty node) and arg [B*M, C] int64: the global sorted row of the value (-1 when empty).
    A node with nothing above the floor takes the reference's index 0: point n = 0 of its cloud."""
    B, N = perm.shape
    M = seg_off.shape[1] - 1
    C = X.shape[1]
    p = perm.long()
    counts = (seg_off[:, 1:] - seg_off[:, :-1]).long()
    node_of_row = torch.repeat_interleave(torch.arange(M, device=X.device).repeat(B), counts.reshape(-1)).view(B, N)
    orig = torch.empty((B, C, N), dtype=X.dtype, device=X.device)
    orig.scatter_(2, p.unsqueeze(1).expand(B, C, N), X.view(B, N, C).permute(0, 2, 1))
    node_of_point = torch.empty((B, N), dtype=torch.int64, device=X.device).scatter_(1, p, node_of_row)
    n = index_max(orig, node_of_point, M)                                    # (B, C, M) original point
    inv = torch.empty_like(p).scatter_(1, p, torch.arange(N, device=X.device).expand(B, N))
    nonempty = (counts > 0).unsqueeze(1)
    pooled = torch.where(nonempty, orig.gather(2, n), torch.zeros((), dtype=X.dtype, device=X.device))
    row = inv.gather(1, n.reshape(B, -1)).view(B, C, M) + torch.arange(B, device=X.device).view(B, 1, 1) * N
    arg = torch.where(nonempty, row, torch.full_like(row, -1))
    return pooled.permute(0, 2, 1).reshape(B * M, C), arg.permute(0, 2, 1).reshape(B * M, C)


def cluster_mean_decenter(xyz, feat, seg_off, perm):
    """networks.py:87-108 in sorted-row order: cluster_mean (B, 3, M) = sum of the node's points / (count + 1e-5), and
    x_aug rows [B*N, 3 + S] = (x - cluster_mean[node], sn) for sorted row r = point perm[b, r]."""
    B, _, N = xyz.shape
    M = seg_off.shape[1] - 1
    p = perm.long()
    counts = (seg_off[:, 1:] - seg_off[:, :-1]).long()
    node = torch.repeat_interleave(torch.arange(M, device=xyz.device).repeat(B), counts.reshape(-1)).view(B, N)
    xs = xyz.gather(2, p.unsqueeze(1).expand(B, 3, N))                         # sorted order
    sums = torch.zeros((B, 3, M), dtype=xyz.dtype, device=xyz.device).scatter_add_(2, node.unsqueeze(1).expand(B, 3, N), xs)
    cmean = sums / (counts.unsqueeze(1).to(xyz.dtype) + 1e-5)
    rows = xs - cmean.gather(2, node.unsqueeze(1).expand(B, 3, N))
    if feat is not None:
        rows = torch.cat([rows, feat.gather(2, p.unsqueeze(1).expand(B, feat.shape[1], N))], 1)
    return cmean, rows.permute(0, 2, 1).reshape(B * N, -1)


def knn_nodes(pts, K):
    """layers.py:417-421: the K nearest nodes of every node by torch.norm distance, ascending, ties by index
    (topk(K, largest=False, sorted=True)); pts (B, 3, M) -> (B, M, K) int64.  Columns K >= M (topk would raise) are 0."""
    M = pts.shape[2]
    d = torch.norm(pts.unsqueeze(3) - pts.unsqueeze(2), dim=1)                # (B, M, M)
    order = torch.sort(d, dim=2, stable=True).indices[:, :, :min(K, M)]
    if K > M:
        order = torch.cat([order, order.new_zeros(order.shape[:2] + (K - M,))], 2)
    return order


def knn_gather(src, idx):
    """operations.py:271-287 knn_gather_by_indexing: out[b, c, m, k] = src[b, c, idx[b, m, k]]."""
    B, C, _ = src.shape
    _, M, K = idx.shape
    return torch.gather(src, 2, idx.long().reshape(B, 1, M * K).expand(B, C, M * K)).view(B, C, M, K)


def desc_pairmin(a, b):
    """DescPairScanLoss's search (losses.py:199-233): for a (B, C, Ma), b (B, C, Nb), torch.norm over C then torch.min
    over the database -> (min_d (B, Ma), arg (B, Ma) int64, the first index on an exact tie)."""
    d = torch.norm(a.unsqueeze(3) - b.unsqueeze(2), dim=1)                    # (B, Ma, Nb)
    mn = d.min(2).values
    j = torch.arange(d.shape[2], device=d.device).expand_as(d)
    return mn, torch.where(d == mn.unsqueeze(2), j, torch.full_like(j, d.shape[2])).min(2).values


def chamfer_prob_terms(d_sd, i_sd, d_ds, i_ds, sig_src, sig_dst):
    """ChamferLoss_Brute's sigma branch (losses.py:79-97) from the two nearest-neighbour searches: sigma of a pair =
    (own sigma + sigma of the nearest point of the other set) / 2, then (loss, chamfer_pure, chamfer_weighted) with
    weights (1/s) / mean(1/s) per direction."""
    s_sd = 0.5 * (sig_src + torch.gather(sig_dst, 1, i_sd.long()))
    s_ds = 0.5 * (sig_dst + torch.gather(sig_src, 1, i_ds.long()))
    loss = (torch.log(s_sd) + d_sd / s_sd).mean() + (torch.log(s_ds) + d_ds / s_ds).mean()
    pure = d_sd.mean() + d_ds.mean()
    w_sd, w_ds = 1 / s_sd, 1 / s_ds
    weighted = (d_sd * w_sd / w_sd.mean()).mean() + (d_ds * w_ds / w_ds.mean()).mean()
    return torch.stack([loss, pure, weighted])
