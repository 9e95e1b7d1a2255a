"""-m gpu: forward entry points of csrc/mlp.cu, csrc/group.cu, csrc/indexmax.cu and csrc/loss.cu, called through the C ABI
at the shapes and layouts where their dispatch changes, against the float64 formulas of tests/forward_ref.py evaluated
on the same GPU (those formulas are checked against the reference's torch expressions by tests/test_forward_refs.py).

Discrete decisions are inputs or are built with a margin: every ReLU argument is >= 1e-3 from 0, nearest neighbours are
separated, and ties come from duplicated values, which give identical fp32 arithmetic.  Kernels whose fp32 operations
can be replayed exactly are compared bit for bit (knn_gather, knn_nodes, segmax values and rows, the decentred rows of
cluster_mean_decenter given the kernel's own mean); group_select is held to 1 ulp of the float64 value.  Everything
else has a tolerance: the comment beside each one gives the worst error measured on an H100 80GB HBM3 (SXM, 700 W power
limit) over the cases of the test, and the tolerance is >= 4x that."""
import ctypes

import numpy as np
import pytest
import torch

from tests import forward_ref as R

pytestmark = pytest.mark.gpu

f32, f64, i32 = torch.float32, torch.float64, torch.int32
NAN = float("nan")
EPS, MOM = float(np.float32(1e-5)), float(np.float32(0.1))     # the fp32 arguments as the kernels widen them


def _lib():
    from usip_b200 import _lib as L
    return L


def P(t, off=0):
    """Device address of tensor t, `off` elements further (None -> NULL)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr() + off * t.element_size())


def call(name, *args):
    from usip_b200.ops import _stream
    L = _lib()
    L.check(getattr(L.load(), name)(*args, _stream()), name)


def dev():
    return torch.device("cuda:0")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(*shape, g, scale=1.0):
    return torch.randn(*shape, generator=g, device=dev(), dtype=f32) * scale


def rand(*shape, g):
    return torch.rand(*shape, generator=g, device=dev(), dtype=f32)


def rel(got, ref):
    """max |got - ref| / max |ref|"""
    ref = ref.double()
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def check(what, err, tol):
    print("measured %-52s %.3e  (tol %.0e)" % (what, err, tol))
    assert err <= tol, (what, err, tol)


def ulps(got, ref):
    """max |got - ref| in units of the fp32 spacing at |ref| (the spacing of the smallest normal below it)."""
    r32 = ref.float().abs().clamp_min(torch.finfo(f32).tiny)
    sp = (torch.nextafter(r32, torch.full_like(r32, float("inf"))) - r32).double()
    return float(((got.double() - ref.double()).abs() / sp).max())


def stat_tiles(Y, rows=128):
    """float64 (sum, sum of squares) of every 128-row tile of Y [G, C] -> [ntiles, 2, C]."""
    G, C = Y.shape
    nt = (G + rows - 1) // rows
    Yp = torch.zeros((nt * rows, C), dtype=f64, device=Y.device)
    Yp[:G] = Y.double()
    t = Yp.view(nt, rows, C)
    return torch.stack([t.sum(1), (t * t).sum(1)], 1)


# ================================================================================ knn_combine
@pytest.mark.parametrize("B,M,K,Cout", [(2, 37, 16, 64),      # G % 128 = 32: tail tile
                                        (1, 50, 8, 192),      # Cout > 128: two channel passes per lane
                                        (3, 64, 16, 256)])
def test_knn_combine(B, M, K, Cout):
    g = gen(B * 1000 + M + Cout)
    Q, G = B * M, B * M * K
    ldz, ldy, ldw = Cout + 12, Cout + 8, 3 + 64
    Z = torch.full((Q, ldz), NAN, device=dev()); Z[:, :Cout] = randn(Q, Cout, g=g)
    pts = randn(B, 3, M, g=g, scale=3.0)
    knn = torch.randint(0, M, (B, M, K), generator=g, device=dev()).to(i32)
    W = torch.full((Cout, ldw), NAN, device=dev()); W[:, :3] = randn(Cout, 3, g=g)
    bias = randn(Cout, g=g, scale=2.0)
    Y = torch.full((G, ldy), NAN, device=dev())
    nt = (G + 127) // 128
    part = torch.full((nt, 2, Cout), NAN, device=dev())
    call("usip_knn_combine", P(Z), ldz, P(pts), P(knn), P(W), ldw, P(bias), P(Y), ldy, P(part), B, M, K, Cout)
    torch.cuda.synchronize()
    ref = R.knn_combine_fwd(Z[:, :Cout].double(), pts.double(), knn, W[:, :3].double(), bias.double())
    tag = "B=%d M=%d K=%d Cout=%d" % (B, M, K, Cout)
    # three fp32 fmas and two adds per element: measured <= 1.1e-7
    check("knn_combine Y " + tag, rel(Y[:, :Cout], ref), 5e-7)
    assert bool(torch.isnan(Y[:, Cout:]).all()), "knn_combine wrote outside [G, Cout]"
    # fp32 partial sums of <= 128 rows per tile: measured <= 2.1e-7 of the tile's sum of |y| / y^2
    st = stat_tiles(Y[:, :Cout])
    mag = stat_tiles(Y[:, :Cout].abs())
    assert not torch.isnan(part).any()
    check("knn_combine stat sums " + tag, float(((part[:, 0].double() - st[:, 0]).abs() / mag[:, 0].clamp_min(1e-30)).max()), 1e-6)
    check("knn_combine stat sumsq " + tag, float(((part[:, 1].double() - st[:, 1]).abs() / mag[:, 1].clamp_min(1e-30)).max()), 1e-6)


# ================================================================================ group_select
@pytest.mark.parametrize("case", ["vec", "odd_offset", "c_not_mult4"])
def test_group_select(case):
    """float4 kernel (C % 4 == 0, aligned rows) and scalar kernel (out = AGG[:, C1:] with C1 odd, or C % 4 != 0); negative,
    +0 and -0 scales.  Held to 1 ulp of the float64 max_k relu(bn(y_k))."""
    Q, K = 333, 8
    C = 30 if case == "c_not_mult4" else 64
    g = gen({"vec": 1, "odd_offset": 2, "c_not_mult4": 3}[case])
    scale = (rand(C, g=g) + 0.25) * torch.where(rand(C, g=g) < 0.4, -1.0, 1.0)
    scale[3], scale[6] = 0.0, -0.0
    shift = randn(C, g=g, scale=0.5)
    Yg = randn(Q, K, C, g=g)
    z = Yg.double() * scale.double() + shift.double()
    Yg = torch.where(z.abs() < 1e-3, Yg + 0.01 * torch.sign(scale + 1e-30), Yg)    # ReLU arguments >= 1e-3 from 0
    gmax, gmin = Yg.amax(1).contiguous(), Yg.amin(1).contiguous()
    off = 5 if case == "odd_offset" else 0
    ldo = off + C + (3 if case == "odd_offset" else 0)
    AGG = torch.full((Q, ldo), NAN, device=dev())
    call("usip_group_select", P(gmax), P(gmin), P(scale), P(shift), P(AGG, off), ldo, Q, C)
    torch.cuda.synchronize()
    ref = R.group_max_relu_bn(Yg.double(), scale.double(), shift.double())
    out = AGG[:, off:off + C]
    assert ulps(out, ref) <= 1.0, ulps(out, ref)
    assert bool(torch.isnan(AGG[:, :off]).all()) and bool(torch.isnan(AGG[:, off + C:]).all())
    neg = scale < 0
    assert bool((ref[:, neg] > 0).any())                # the negative-scale channels have live outputs: the min was picked


# ================================================================================ BatchNorm finalize / eval
@pytest.mark.parametrize("ntiles,C", [(1, 8), (20, 12), (300, 64), (333, 13), (2049, 40)])
def test_bn_finalize(ntiles, C):
    """Fixed-order float64 sum of the partial rows: one batch, a tail batch (ntiles not a multiple of 256, and < 32),
    C % 8 != 0; with and without gamma / beta, save_mean / save_invstd and running statistics."""
    g = gen(ntiles * 100 + C)
    count = 1 if ntiles == 1 else ntiles * 128 - 37
    rows = randn(ntiles, 128, C, g=g, scale=2.0) + randn(1, 1, C, g=g, scale=3.0)
    part = torch.stack([rows.sum(1), (rows * rows).sum(1)], 1).contiguous()     # any fp32 partials will do
    S, SS = part[:, 0].double().sum(0), part[:, 1].double().sum(0)
    gamma, beta = rand(C, g=g) + 0.5, randn(C, g=g)
    rm0, rv0 = randn(C, g=g), rand(C, g=g) + 0.5
    for affine in (True, False):
        rm, rv = rm0.clone(), rv0.clone()
        scale, shift = torch.full((C,), NAN, device=dev()), torch.full((C,), NAN, device=dev())
        sm, si = torch.full((C,), NAN, device=dev()), torch.full((C,), NAN, device=dev())
        call("usip_bn_finalize", P(part), ntiles, count, C, P(gamma) if affine else None, P(beta) if affine else None,
             1e-5, 0.1, P(rm), P(rv), P(scale), P(shift), P(sm), P(si))
        torch.cuda.synchronize()
        r_scale, r_shift, r_mean, r_inv, r_rm, r_rv = R.bn_train_from_sums(
            S, SS, count, gamma.double() if affine else None, beta.double() if affine else None, EPS, MOM,
            rm0.double(), rv0.double())
        tag = "ntiles=%d C=%d affine=%d" % (ntiles, C, affine)
        # a float64 sum of the same fp32 partials, then one fp32 rounding: measured <= 0.50 ulp
        for nm, got, ref in (("scale", scale, r_scale), ("mean", sm, r_mean), ("invstd", si, r_inv),
                             ("running_mean", rm, r_rm), ("running_var", rv, r_rv)):
            check("bn_finalize %s %s" % (nm, tag), ulps(got, ref), 2.0)
        # shift = beta - mean * scale rounds once in fp32 from a float64 difference: measured <= 4.1e-8
        check("bn_finalize shift " + tag, float(((shift.double() - r_shift).abs() /
                                                 (r_shift.abs() + (r_mean * r_scale).abs())).max()), 2.4e-7)
    # the same call without the optional outputs writes scale / shift alone
    s2, h2 = torch.empty(C, device=dev()), torch.empty(C, device=dev())
    call("usip_bn_finalize", P(part), ntiles, count, C, P(gamma), P(beta), 1e-5, 0.1, None, None, P(s2), P(h2), None, None)
    torch.cuda.synchronize()
    r_scale, r_shift, *_ = R.bn_train_from_sums(S, SS, count, gamma.double(), beta.double(), EPS, MOM)
    assert ulps(s2, r_scale) <= 2.0


@pytest.mark.parametrize("ratio", [0, 10, 30, 100])
def test_bn_finalize_large_mean(ratio):
    """Statistics of real rows through the SIMT layer's fp32 tile partials (sum and fma sum of squares): the variance is
    E[y^2] - E[y]^2, so its error grows with |mean| / std.  Identity weights make Y == X exactly."""
    Pn, C = 65536 + 37, 16
    g = gen(ratio + 7)
    X = randn(Pn, C, g=g) + ratio * torch.where(torch.arange(C, device=dev()) % 2 == 0, 1.0, -1.0)
    W = torch.eye(C, device=dev())
    from usip_b200 import ops
    nt = (Pn + 127) // 128
    part = torch.full((nt, 2, C), NAN, device=dev())
    Y = torch.empty_like(X)
    ops.layer_fwd(X, W, None, Pn, C, C, Y=Y, stat_partial=part)
    scale, shift = torch.empty(C, device=dev()), torch.empty(C, device=dev())
    sm, si = torch.empty(C, device=dev()), torch.empty(C, device=dev())
    ops.bn_finalize(part, nt, Pn, C, None, None, 1e-5, 0.1, None, None, scale, shift, sm, si)
    torch.cuda.synchronize()
    assert torch.equal(Y, X)
    Xd = X.double()
    ref_inv = 1.0 / torch.sqrt(Xd.var(0, unbiased=False) + 1e-5)
    err = rel(si, ref_inv)
    # measured <= 1.0e-7
    check("bn_finalize mean |mean|/std=%d" % ratio, rel(sm, Xd.mean(0)), 5e-7)
    # the bound of usip_b200.h, 2.5e-7 + 4e-8 (|mean|/std)^2; measured 5.8e-8, 8.1e-7, 4.5e-6 and 6.2e-5 at 0, 10, 30, 100
    check("bn_finalize invstd |mean|/std=%d" % ratio, err, 2.5e-7 + 4e-8 * ratio ** 2)


def test_bn_eval_affine():
    C = 333
    g = gen(21)
    gamma, beta, rm, rv = randn(C, g=g), randn(C, g=g), randn(C, g=g, scale=3.0), rand(C, g=g) * 4 + 1e-4
    scale, shift = torch.full((C,), NAN, device=dev()), torch.full((C,), NAN, device=dev())
    call("usip_bn_eval_affine", P(gamma), P(beta), P(rm), P(rv), 1e-5, C, P(scale), P(shift))
    torch.cuda.synchronize()
    r_scale, r_shift = R.bn_eval(gamma.double(), beta.double(), rm.double(), rv.double(), EPS)
    # fp32 1/sqrtf and one product: measured <= 1.33 ulp
    check("bn_eval scale (ulp)", ulps(scale, r_scale), 6.0)
    # measured <= 1.2e-7 of |beta| + |mean scale|
    check("bn_eval shift", float(((shift.double() - r_shift).abs() / (beta.double().abs() + (rm.double() * r_scale).abs())).max()), 1e-6)


# ================================================================================ narrow layers
@pytest.mark.parametrize("Cout", [4, 8])
def test_layer_fwd_rowwarp_prologue_transposed(Cout):
    """The one-warp-per-row kernel (Cout <= 8) with the BN + ReLU prologue and a transposed weight [Cin, Cout]."""
    from usip_b200 import ops
    Pn, Cin = 1000, 256
    g = gen(Cout)
    X = randn(Pn, Cin + 4, g=g)
    Wt = torch.full((Cin, Cout + 3), NAN, device=dev()); Wt[:, :Cout] = randn(Cin, Cout, g=g, scale=Cin ** -0.5)
    b, sc, sh = randn(Cout, g=g), randn(Cin, g=g), randn(Cin, g=g)
    Y = torch.full((Pn, Cout + 2), NAN, device=dev())
    ops.layer_fwd(X, Wt, b, Pn, Cin, Cout, ldx=Cin + 4, ldw=Cout + 3, in_scale=sc, in_shift=sh, in_relu=True,
                  Y=Y, ldy=Cout + 2, w_transposed=True)
    torch.cuda.synchronize()
    ref = R.layer_fwd(X[:, :Cin].double(), Wt[:, :Cout].double().t(), b.double(), sc.double(), sh.double(), True)
    # fp32 fma chains over Cin/32 terms per lane and a warp tree: measured <= 1.2e-7
    check("layer_fwd rowwarp Cout=%d" % Cout, rel(Y[:, :Cout], ref), 5e-7)
    assert bool(torch.isnan(Y[:, Cout:]).all())


@pytest.mark.parametrize("Cout", [32, 64])
@pytest.mark.parametrize("layout", ["ldx3", "unaligned"])
def test_layer_fwd_narrow_scalar_load(Cout, layout):
    """The first-layer kernel (Cin <= 8, Cout 32 / 64) reading X with scalar loads: ldx < 8, or X one float off a 16-byte
    boundary; Y and the statistics partials of every 128-row tile."""
    from usip_b200 import ops
    Pn, Cin = 1000, 3
    g = gen(Cout + len(layout))
    if layout == "ldx3":
        ldx, buf, off = 3, randn(Pn, 3, g=g), 0
    else:
        ldx, buf, off = 8, randn(Pn * 8 + 1, g=g), 1
    X = buf.view(-1)[off:off + (Pn - 1) * ldx + Cin].as_strided((Pn, Cin), (ldx, 1))
    W, b = randn(Cout, Cin, g=g), randn(Cout, g=g)
    Y = torch.full((Pn, Cout), NAN, device=dev())
    nt = (Pn + 127) // 128
    part = torch.full((nt, 2, Cout), NAN, device=dev())
    d = _lib().LayerDesc()
    d.X = X.data_ptr(); d.ldx = ldx; d.P = Pn; d.Cin = Cin; d.Cout = Cout
    d.W = W.data_ptr(); d.ldw = Cin; d.bias = b.data_ptr(); d.Y = Y.data_ptr(); d.ldy = Cout
    d.stat_partial = part.data_ptr()
    from usip_b200.ops import _stream
    _lib().check(_lib().load().usip_layer_fwd(ctypes.byref(d), _stream()), "usip_layer_fwd")
    torch.cuda.synchronize()
    ref = R.layer_fwd(X.double(), W.double(), b.double())
    # <= 4 fp32 fmas per element: measured <= 9.2e-8; tile statistics: measured <= 1.9e-7 of sum |y| / y^2
    check("layer_fwd narrow %s Cout=%d" % (layout, Cout), rel(Y, ref), 5e-7)
    st, mag = stat_tiles(ref), stat_tiles(ref.abs())
    check("layer_fwd narrow stats %s Cout=%d" % (layout, Cout),
          float(((part.double() - st).abs() / mag.clamp_min(1e-30)).max()), 1e-6)


# ================================================================================ grouping front-end
def _nodes(B, N, M, g, empty=(), big=None):
    """A random node per point (some nodes empty, one node `big` holding a third of the points) -> seg_off, perm."""
    node = torch.randint(0, M, (B, N), generator=g, device=dev())
    if big is not None:
        node[:, : N // 3] = big
    for m in empty:
        node[node == m] = (m + 1) % M
    perm = torch.sort(node, dim=1, stable=True).indices
    counts = torch.stack([torch.bincount(r, minlength=M) for r in node])
    seg = torch.cat([torch.zeros(B, 1, dtype=torch.int64, device=dev()), counts.cumsum(1)], 1)
    return node, seg.to(i32).contiguous(), perm.to(i32).contiguous(), counts


@pytest.mark.parametrize("C", [64, 96, 200])
def test_segmax(C):
    """Half-warp kernel (C <= 64) and the lane loop (C > 64): exact ties on adjacent sorted rows (split across the two
    half-warps), values at and below the -1000 floor, a node with nothing above it (falls back to point 0 of its cloud),
    NaN, empty nodes, strided X and pooled."""
    B, N, M = 2, 3000, 40
    g = gen(C)
    node, seg, perm, counts = _nodes(B, N, M, g, empty=(5, 17), big=9)
    ldx, ldp = C + 4, C + 8
    X = torch.full((B * N, ldx), NAN, device=dev()); X[:, :C] = randn(B * N, C, g=g)
    Xv = X[:, :C].view(B, N, C)
    so = seg.long().cpu()
    for b in range(B):
        for m in range(M):
            s, e = int(so[b, m]), int(so[b, m + 1])
            if e - s >= 3:
                Xv[b, s, 0::3] = Xv[b, s + 1, 0::3] = 5.0 + m          # first maximum on an even row, tie on the next
                Xv[b, s + 1, 1::3] = Xv[b, s + 2, 1::3] = 6.0 + m      # first maximum on an odd row
    m0 = int(node[0, 0])                                              # the node of point 0 of cloud 0
    s0, e0 = int(so[0, m0]), int(so[0, m0 + 1])
    Xv[0, s0:e0, 2] = -2000.0
    Xv[0, s0:e0:2, 2] = -1000.0                                       # exactly the floor is not above it
    Xv[1, int(so[1, 3]):int(so[1, 4]), 4] = -1000.0
    Xv[:, 7::11, 5] = NAN
    pooled = torch.full((B * M, ldp), NAN, device=dev())
    arg = torch.full((B * M, C), -7, dtype=i32, device=dev())
    call("usip_segmax", P(X), ldx, P(seg), P(perm), P(pooled), ldp, P(arg), B, N, M, C)
    torch.cuda.synchronize()
    r_pool, r_arg = R.segmax(X[:, :C].double(), seg.long(), perm.long())
    assert torch.equal(arg.long(), r_arg), int((arg.long() != r_arg).sum())
    assert torch.equal(pooled[:, :C].double(), r_pool)
    assert bool(torch.isnan(pooled[:, C:]).all())
    assert bool((arg.view(B, M, C)[:, 5] == -1).all()) and bool((pooled[:, :C].reshape(B, M, C)[:, 17] == 0).all())


@pytest.mark.parametrize("S,ldx", [(0, 3), (0, 8), (4, 11), (7, 12)])
def test_cluster_mean_decenter(S, ldx):
    """The scalar path (ldx != 8 or S > 5), the vector path at S = 0, an empty node: the decentred rows are compared bit
    for bit against fl32(x - the kernel's own mean), the features and zero padding exactly, the mean with a tolerance."""
    B, N, M = 2, 2000, 50
    g = gen(S * 100 + ldx)
    xyz, sn = randn(B, 3, N, g=g, scale=5.0), randn(B, S, N, g=g) if S else None
    _, seg, perm, counts = _nodes(B, N, M, g, empty=(8,))
    cmean = torch.full((B, 3, M), NAN, device=dev())
    x_aug = torch.full((B * N, ldx), NAN, device=dev())
    call("usip_cluster_mean_decenter", P(xyz), P(sn), P(seg), P(perm), P(cmean), P(x_aug), ldx, B, S, N, M)
    torch.cuda.synchronize()
    r_mean, r_rows = R.cluster_mean_decenter(xyz.double(), None if sn is None else sn.double(), seg.long(), perm.long())
    # fp32 lane sums and a warp tree: measured <= 1.6e-8 of max |x|
    check("cluster_mean S=%d ldx=%d" % (S, ldx), float((cmean.double() - r_mean).abs().max() / xyz.abs().max()), 1e-7)
    assert bool((cmean[:, :, 8] == 0).all())
    p = perm.long()
    xs = xyz.gather(2, p.unsqueeze(1).expand(B, 3, N))
    counts_ = counts.to(dev())
    node_sorted = torch.repeat_interleave(torch.arange(M, device=dev()).repeat(B), counts_.reshape(-1)).view(B, N)
    dec = (xs - cmean.gather(2, node_sorted.unsqueeze(1).expand(B, 3, N))).permute(0, 2, 1).reshape(B * N, 3)
    assert torch.equal(x_aug[:, :3], dec)
    if S:
        assert torch.equal(x_aug[:, 3:3 + S], r_rows[:, 3:].float())
    assert bool((x_aug[:, 3 + S:] == 0).all())


@pytest.mark.parametrize("B,C,N,M,K", [(2, 1, 100, 7, 3),        # C = 1, 42 outputs per cloud
                                       (3, 5, 50, 13, 1),        # K = 1
                                       (2, 64, 300, 37, 16)])    # B*C*M*K = 75776, not a multiple of 256
def test_knn_gather(B, C, N, M, K):
    g = gen(B + C + N)
    src = randn(B, C, N, g=g)
    idx = torch.randint(0, N, (B, M, K), generator=g, device=dev()).to(i32)
    out = torch.full((B, C, M, K), NAN, device=dev())
    call("usip_knn_gather_f32", P(src), P(idx), P(out), B, C, N, M, K)
    torch.cuda.synchronize()
    assert torch.equal(out, R.knn_gather(src, idx))


# ================================================================================ index_max with offset operands
@pytest.mark.parametrize("B,C,N,K", [(2, 64, 2048, 64),          # the bucket kernel's shape
                                     (1, 4, 1024, 10)])          # the shared-memory atomic kernel's shape
def test_index_max_unaligned_operands(B, C, N, K):
    """forward_cuda_shared_mem with data and / or index one element past a 16-byte boundary (contiguous views into a
    larger buffer), N % 4 == 0: the 16-byte loads must not be taken, the result must not change."""
    from oracle import usip_oracle as orc
    from usip_b200 import index_max
    g = gen(B * C + N)
    dbuf = randn(B * C * N + 4, g=g)
    ibuf = torch.randint(0, K, (B * N + 4,), generator=g, device=dev()).to(i32)
    for doff, ioff in ((0, 0), (1, 0), (0, 1), (1, 3)):
        data = dbuf[doff:doff + B * C * N].view(B, C, N)
        index = ibuf[ioff:ioff + B * N].view(B, N)
        out = index_max.forward_cuda_shared_mem(data, index, K)
        torch.cuda.synchronize()
        exp = orc.index_max(data.cpu().numpy(), index.cpu().numpy(), K)
        assert np.array_equal(out.cpu().numpy(), exp), (doff, ioff)


# ================================================================================ losses
@pytest.mark.parametrize("B,M,N", [(4, 1500, 1100),    # B*max(M, N) = 6000: several four-element batches per thread
                                   (1, 600, 50)])      # B*max(M, N) < 1024, M > N
def test_chamfer_prob_reduce_sigma_pairing(B, M, N):
    """M != N with skewed neighbours: every src point's nearest dst point is one of eight with a large sigma, so the two
    directions' mean(1/s) differ by a factor ~5 and a sigma read from the wrong array or a term divided by the other
    direction's mean shows.  Also usip_mean_scale over the same distances."""
    g = gen(B * M + N)
    d_sd, d_ds = rand(B, M, g=g) * 2, rand(B, N, g=g) * 2
    i_sd = torch.randint(0, 8, (B, M), generator=g, device=dev()).to(i32)
    i_ds = torch.randint(0, M, (B, N), generator=g, device=dev()).to(i32)
    ss, sd = rand(B, M, g=g) + 0.2, rand(B, N, g=g) + 0.2
    sd[:, :8] = 8.0 + rand(B, 8, g=g)
    out3 = torch.full((3,), NAN, device=dev())
    call("usip_chamfer_prob_reduce", P(d_sd), P(i_sd), P(d_ds), P(i_ds), P(ss), P(sd), P(out3), B, M, N)
    ms = torch.full((1,), NAN, device=dev())
    call("usip_mean_scale", P(d_sd), B * M, ctypes.c_float(0.37), P(ms))
    torch.cuda.synchronize()
    ref = R.chamfer_prob_terms(d_sd.double(), i_sd, d_ds.double(), i_ds, ss.double(), sd.double())
    # fp32 per-element terms, float64 sums: measured <= 4.9e-8
    check("chamfer_prob_reduce B=%d M=%d N=%d" % (B, M, N), float(((out3.double() - ref).abs() / ref.abs()).max()), 2e-7)
    # a float64 sum, one fp32 rounding, one fp32 product: measured <= 0.58 ulp
    check("mean_scale n=%d (ulp)" % (B * M), ulps(ms, (d_sd.double().mean() * np.float32(0.37)).view(1)), 2.5)


@pytest.mark.parametrize("B,C,Ma,Nb", [(2, 32, 45, 70),        # small C (static shared memory), Ma % 32, Nb % 64 != 0
                                       (1, 128, 300, 7),       # C >= 107: the opt-in attribute, Ma > 256, Nb < 8
                                       (2, 128, 33, 130),      # duplicated database columns
                                       (1, 533, 40, 64)])      # the largest C under the 200 KB limit
def test_desc_pairmin(B, C, Ma, Nb):
    """Every query sits near one database column (a clear nearest neighbour); a duplicated column ties exactly and the
    first index must win."""
    g = gen(C * 7 + Ma)
    b = randn(B, C, Nb, g=g)
    near = torch.randint(0, Nb, (B, Ma), generator=g, device=dev())
    if Nb >= 100:
        b[:, :, Nb - 1] = b[:, :, 5]                                    # column Nb-1 duplicates column 5
        near[:, ::3] = Nb - 1                                           # queries near the duplicate: index 5 must win
    a = (R._col_gather(b, near) + randn(B, C, Ma, g=g, scale=0.01)).contiguous()
    md, arg = torch.full((B, Ma), NAN, device=dev()), torch.full((B, Ma), -7, dtype=i32, device=dev())
    call("usip_desc_pairmin_f32", P(a), P(b), P(md), P(arg), B, C, Ma, Nb)
    torch.cuda.synchronize()
    r_d, r_arg = R.desc_pairmin(a.double(), b.double())
    assert torch.equal(arg.long(), r_arg)
    if Nb >= 100:
        assert bool((arg[:, ::3] == 5).all())
    # fp32 fma chain over C terms of (a - b)^2, then sqrtf: measured <= 3.5e-7
    check("desc_pairmin B=%d C=%d Ma=%d Nb=%d" % (B, C, Ma, Nb), rel(md, r_d), 2e-6)


def test_desc_triplet_zero_weights_and_long_rows():
    """M > 256 (several rows per thread), and a batch whose weights are all zero: w / mean(w) is 0/0 there, NaN as in the
    reference's expression."""
    B, M = 2, 700
    g = gen(31)
    dpos, dneg = rand(B, M, g=g) * 2, rand(B, M, g=g) * 2
    h = dpos.double() - dneg.double() + 0.5
    dpos = torch.where(h.abs() < 1e-3, dpos + 0.01, dpos)
    sigma = rand(B, M, g=g) * 2.5
    sigma[1] = 3.0 + rand(M, g=g)                                      # >= sigma_max everywhere: all weights 0
    loss, active = torch.empty(B, M, device=dev()), torch.empty(B, device=dev())
    call("usip_desc_triplet", P(dpos), P(dneg), P(sigma), ctypes.c_float(0.5), ctypes.c_float(3.0), P(loss), P(active), B, M)
    torch.cuda.synchronize()
    l_ref, a_ref = R.desc_triplet_fwd(dpos.double(), dneg.double(), sigma.double(), 0.5, 3.0)
    assert bool(torch.isnan(l_ref[1]).all()) and bool(torch.isnan(loss[1]).all())
    # measured <= 8.7e-8
    check("desc_triplet loss M=%d" % M, rel(loss[0], l_ref[0]), 5e-7)
    assert torch.equal(active, a_ref.float())
