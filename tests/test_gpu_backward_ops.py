"""-m gpu: every backward entry point of csrc/backward.cu, the loss backward kernels of csrc/loss.cu and usip_adam_step,
called through the C ABI at the shapes and layouts where their dispatch changes, against the float64 formulas of
tests/backward_ref.py evaluated on the same GPU (those formulas are checked against torch.autograd by
tests/test_backward_refs.py).

Discrete decisions are inputs (arg-max rows, neighbour indices) or are built with a margin of >= 1e-3 (every ReLU /
hinge argument), plus deliberate exact zeros, so the comparisons can be tight.  Kernels that do the same fp32 operations
in the same order as a plain fp32 loop (group_sum, seg_sum, unpool_scatter, groupmax_scatter_add, gz / argsel of the
group-max select) are compared bit for bit.  Everything else has a tolerance: the comment beside each one gives the worst
error measured on an H100 80GB HBM3 (SXM, 700 W power limit) over the cases of the test, and the tolerance is >= 4x that."""
import ctypes

import numpy as np
import pytest
import torch

from tests import backward_ref as R

pytestmark = pytest.mark.gpu

f32, f64, i32 = torch.float32, torch.float64, torch.int32
NAN = float("nan")


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


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


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


def red(got, ref, mag):
    """error of a sum relative to the sum of the magnitudes of its terms (max over channels)"""
    return float((got.double() - ref.double()).abs().max() / mag.double().max().clamp_min(1e-30))


def check(what, err, tol):
    print("measured %-44s %.3e  (tol %.0e)" % (what, err, tol))
    assert err <= tol, (what, err, tol)


def with_margin(y, scale, shift, margin=2e-3):
    """Move every y whose pre-activation y*scale + shift lies within `margin` of 0 to pre-activation 0.01."""
    z = y.double() * scale.double() + shift.double()
    fix = ((0.01 - shift.double()) / scale.double()).float().expand_as(y)
    return torch.where(z.abs() < margin, fix, y)


# ================================================================================ BatchNorm backward
def big_p():
    """Ragged row count above 4 * SMs * 128, where the reduce kernel's CTAs loop over tiles and leave partial rows to zero."""
    return 4 * sm_count() * 128 + 1000 + 37


def bn_inputs(Pn, C, seed, pad=8):
    g = gen(seed)
    ld = C + pad
    G = torch.full((Pn, ld), NAN, device=dev()); G[:, :C] = randn(Pn, C, g=g)
    Y = torch.full((Pn, ld), NAN, device=dev())
    scale = (rand(C, g=g) + 0.5) * torch.where(rand(C, g=g) < 0.35, -1.0, 1.0)
    shift = randn(C, g=g, scale=0.5)
    shift[1] = 0.0
    mean = randn(C, g=g, scale=0.1)
    invstd = rand(C, g=g) + 0.5
    y = with_margin(randn(Pn, C, g=g), scale, shift)
    y[::7, 1] = 0.0                                     # y = 0, shift = 0: pre-activation exactly 0, ReLU closed
    Y[:, :C] = y
    return G, Y, scale, shift, mean, invstd


@pytest.mark.parametrize("C", [32, 64, 128, 256, 512, 48, 96])       # 48, 96: tile reduce + generic apply kernels
@pytest.mark.parametrize("rows", ["1", "127", "129", "big"])
def test_bn_bwd_reduce_finalize_apply(C, rows):
    Pn = big_p() if rows == "big" else int(rows)
    G, Y, scale, shift, mean, invstd = bn_inputs(Pn, C, seed=C * 7 + Pn)
    ld = G.shape[1]
    nt = (Pn + 127) // 128
    for relu in (1, 0):
        part = torch.full((nt, 2, C), NAN, device=dev())               # every partial row must be written
        call("usip_bn_bwd_reduce", P(G), ld, P(Y), ld, P(scale), P(shift), P(mean), P(invstd), relu, P(part), Pn, C)
        gg = torch.empty(C, device=dev()); gb = torch.empty(C, device=dev())
        c1 = torch.empty(C, device=dev()); c2 = torch.empty(C, device=dev())
        call("usip_bn_bwd_finalize", P(part), nt, Pn, C, P(gg), P(gb), P(c1), P(c2), 0)
        ldo = C + 12
        GY = torch.full((Pn, ldo), 7.0, device=dev())
        call("usip_bn_bwd_apply", P(G), ld, P(Y), ld, P(scale), P(shift), P(mean), P(invstd), P(c1), P(c2), relu, P(GY), ldo, Pn, C)
        Gi = G.clone()                                                 # in place: GY aliases G
        call("usip_bn_bwd_apply", P(Gi), ld, P(Y), ld, P(scale), P(shift), P(mean), P(invstd), P(c1), P(c2), relu, P(Gi), ld, Pn, C)
        torch.cuda.synchronize()

        g64, y64 = G[:, :C].double(), Y[:, :C].double()
        gy_ref, gg_ref, gb_ref = R.bn_relu_bwd(g64, y64, scale.double(), shift.double(), mean.double(), invstd.double(), relu)
        gz = g64 * ((y64 * scale.double() + shift.double()) > 0) if relu else g64
        xhat = (y64 - mean.double()) * invstd.double()
        mag_b, mag_g = gz.abs().sum(0), (gz * xhat).abs().sum(0)
        ps = part.double().sum(0)
        assert not torch.isnan(part).any()
        tag = "C=%d P=%d relu=%d" % (C, Pn, relu)
        # fp32 partial sums over at most P/(4*SMs) rows per thread, then a float64 finalize: measured <= 1.1e-7 of sum|term|
        check("bn reduce g_beta " + tag, red(ps[0], gb_ref, mag_b), 5e-7)
        check("bn reduce g_gamma " + tag, red(ps[1], gg_ref, mag_g), 5e-7)
        check("bn finalize g_beta " + tag, red(gb, gb_ref, mag_b), 5e-7)
        check("bn finalize g_gamma " + tag, red(gg, gg_ref, mag_g), 5e-7)
        # per element: a handful of fp32 roundings of O(1) terms; measured <= 2.0e-7 of max|g_y|
        check("bn apply g_y " + tag, rel(GY[:, :C], gy_ref), 1e-6)
        assert bool((GY[:, C:] == 7.0).all()), "apply wrote outside [P, C]"
        assert torch.equal(Gi[:, :C], GY[:, :C]), "in-place apply differs from out-of-place"
        assert bool(torch.isnan(Gi[:, C:]).all())


@pytest.mark.parametrize("ntiles", [1, 20, 300, 333])
def test_bn_bwd_finalize(ntiles):
    """Fixed-order float64 sum of the partial rows: g_beta / g_gamma written or accumulated, NULL outputs, c1 / c2."""
    C, count = 44, 98765
    g = gen(ntiles)
    part = randn(ntiles, 2, C, g=g)
    A, B = part[:, 0].double().sum(0), part[:, 1].double().sum(0)
    eps = 2.0 ** -23
    for acc in (0, 1):
        gb0, gg0 = randn(C, g=g), randn(C, g=g)
        gb, gg = gb0.clone(), gg0.clone()
        c1 = torch.full((C,), NAN, device=dev()); c2 = torch.full((C,), NAN, device=dev())
        call("usip_bn_bwd_finalize", P(part), ntiles, count, C, P(gg), P(gb), P(c1), P(c2), acc)
        torch.cuda.synchronize()
        base_b, base_g = (gb0.double(), gg0.double()) if acc else (0.0, 0.0)
        # two fp32 roundings (the float64 sum, then the add): <= 2 ulp of the operands
        assert bool(((gb.double() - (base_b + A)).abs() <= 2 * eps * (abs(base_b) + A.abs()) + 1e-30).all()), acc
        assert bool(((gg.double() - (base_g + B)).abs() <= 2 * eps * (abs(base_g) + B.abs()) + 1e-30).all()), acc
        assert bool(((c1.double() - A / count).abs() <= eps * (A / count).abs()).all())
        assert bool(((c2.double() - B / count).abs() <= eps * (B / count).abs()).all())
    c1n = torch.full((C,), NAN, device=dev()); c2n = torch.full((C,), NAN, device=dev())
    call("usip_bn_bwd_finalize", P(part), ntiles, count, C, None, None, P(c1n), P(c2n), 1)
    torch.cuda.synchronize()
    assert torch.equal(c1n, c1) and torch.equal(c2n, c2)


# ================================================================================ group max
def groupmax_inputs(K, Q, C, seed):
    g = gen(seed)
    y = randn(Q, K, C, g=g)
    kmax = torch.randint(0, K, (Q, C), generator=g, device=dev())
    kmin = (kmax + 1 + torch.randint(0, K - 1, (Q, C), generator=g, device=dev())) % K
    top, bot = y.amax(1), y.amin(1)
    y.scatter_(1, kmax.unsqueeze(1), (top + 0.25).unsqueeze(1))       # unique maximum / minimum of every group
    y.scatter_(1, kmin.unsqueeze(1), (bot - 0.25).unsqueeze(1))
    scale = (rand(C, g=g) + 0.5) * torch.where(rand(C, g=g) < 0.4, -1.0, 1.0)
    scale[2] = 0.0; scale[5] = 0.0                                     # scale exactly 0: the gmax branch, z = shift
    shift = randn(C, g=g, scale=0.5)
    shift[2], shift[5] = 0.7, -0.7
    # margin of the selected pre-activation: push the selected value further out (keeps it the max / min)
    sel = torch.where(scale >= 0, kmax, kmin)
    ysel = y.gather(1, sel.unsqueeze(1)).squeeze(1)
    z = ysel.double() * scale.double() + shift.double()
    bump = torch.where(z.abs() < 2e-3, 0.01 * torch.sign(scale).double(), torch.zeros_like(z)).float()
    y.scatter_(1, sel.unsqueeze(1), (ysel + bump).unsqueeze(1))
    gmax, gmin = y.amax(1), y.amin(1)
    assert torch.equal(y.argmax(1), kmax) and torch.equal(y.argmin(1), kmin)
    mean = randn(C, g=g, scale=0.1)
    invstd = rand(C, g=g) + 0.5
    return y.view(Q * K, C), gmax, gmin, kmax.to(i32), kmin.to(i32), scale, shift, mean, invstd


@pytest.mark.parametrize("K,Q,C", [(16, 300, 44), (32, 129, 72), (64, 77, 36)])
def test_groupmax_bwd_select_finalize_apply(K, Q, C):
    Yd, gmax, gmin, amax, amin, scale, shift, mean, invstd = groupmax_inputs(K, Q, C, seed=K + Q + C)
    g = gen(3 * Q)
    ldg = C + 5
    Gout = torch.full((Q, ldg), NAN, device=dev()); Gout[:, :C] = randn(Q, C, g=g)
    nt = (Q + 127) // 128
    gz = torch.full((Q, C), NAN, device=dev()); argsel = torch.full((Q, C), -7, dtype=i32, device=dev())
    part = torch.full((nt, 2, C), NAN, device=dev())
    call("usip_groupmax_bwd_select", P(Gout), ldg, P(gmax), P(gmin), P(amax), P(amin), P(scale), P(shift), P(mean),
         P(invstd), P(gz), P(argsel), P(part), Q, C)
    # the variant without statistics (part, mean, invstd NULL) writes the same gz / argsel
    gz2 = torch.full((Q, C), NAN, device=dev()); arg2 = torch.full((Q, C), -7, dtype=i32, device=dev())
    call("usip_groupmax_bwd_select", P(Gout), ldg, P(gmax), P(gmin), P(amax), P(amin), P(scale), P(shift), None, None,
         P(gz2), P(arg2), None, Q, C)
    gg = torch.empty(C, device=dev()); gb = torch.empty(C, device=dev())
    c1 = torch.empty(C, device=dev()); c2 = torch.empty(C, device=dev())
    call("usip_bn_bwd_finalize", P(part), nt, Q * K, C, P(gg), P(gb), P(c1), P(c2), 0)
    ldy = C + 4
    Y = torch.full((Q * K, ldy), NAN, device=dev()); Y[:, :C] = Yd
    ldo = C + 8
    GY = torch.full((Q * K, ldo), 7.0, device=dev())
    call("usip_groupmax_bwd_apply", P(Y), ldy, P(gz), P(argsel), P(scale), P(mean), P(invstd), P(c1), P(c2), P(GY), ldo,
         K, Q * K, C)
    torch.cuda.synchronize()

    gy_ref, gg_ref, gb_ref, gz_ref, as_ref = R.groupmax_bwd(Gout[:, :C].double(), Yd.double(), amax, amin, scale.double(),
                                                            mean.double(), invstd.double(), shift.double())
    assert torch.equal(argsel, as_ref.to(i32)) and torch.equal(arg2, argsel)
    assert torch.equal(gz, gz_ref.float()) and torch.equal(gz2, gz)              # a masked copy of Gout: exact
    assert not torch.isnan(part).any()
    ysel = Yd.view(Q, K, C).gather(1, as_ref.unsqueeze(1)).squeeze(1).double()
    xhat = (ysel - mean.double()) * invstd.double()
    ps = part.double().sum(0)
    tag = "K=%d Q=%d C=%d" % (K, Q, C)
    # sums over <= 128 rows per partial: measured <= 2.9e-8 of sum|term|
    check("groupmax part g_beta " + tag, red(ps[0], gb_ref, gz_ref.abs().sum(0)), 2e-7)
    check("groupmax part g_gamma " + tag, red(ps[1], gg_ref, (gz_ref * xhat).abs().sum(0)), 2e-7)
    # per element, like the BN apply: measured <= 7.0e-8
    check("groupmax apply g_y " + tag, rel(GY[:, :C], gy_ref), 5e-7)
    assert bool((GY[:, C:] == 7.0).all())
    zero = (scale == 0)
    assert bool((GY[:, :C][:, zero] == 0).all())                       # scale 0: no gradient reaches y

    # scatter_add: G[(q*K + argsel), c] += gsrc[q, c], one fp32 add per target
    ldG = C + 3
    Gd = randn(Q * K, ldG, g=g)
    ref = Gd.clone()
    gsrc = randn(Q, C, g=g)
    call("usip_groupmax_scatter_add", P(Gd), ldG, P(gsrc), P(argsel), K, Q, C)
    rows = (torch.arange(Q, device=dev()).view(Q, 1) * K + argsel.long())
    ref[:, :C].scatter_add_(0, rows, gsrc)
    torch.cuda.synchronize()
    assert torch.equal(Gd, ref)


# ================================================================================ group_sum / seg_sum / unpool
def _seq_sum(rows_list):
    acc = torch.zeros_like(rows_list[0])
    for r in rows_list:
        acc = acc + r
    return acc


@pytest.mark.parametrize("K,Q,C", [(16, 100, 64), (32, 37, 136), (4, 5, 4)])
def test_group_sum_bit_exact(K, Q, C):
    g = gen(K * Q + C)
    ldg, ldo = C + 8, C + 4
    G = randn(Q * K, ldg, g=g)
    out = torch.full((Q, ldo), 7.0, device=dev())
    call("usip_group_sum", P(G), ldg, P(out), ldo, K, Q, C)
    torch.cuda.synchronize()
    ref = _seq_sum([G.view(Q, K, ldg)[:, k, :C] for k in range(K)])   # fp32, k ascending: the kernel's order
    assert torch.equal(out[:, :C], ref) and bool((out[:, C:] == 7.0).all())


@pytest.mark.parametrize("C", [64, 136])                               # 136: more float4 groups than lanes
def test_seg_sum_bit_exact(C):
    B, N, M = 2, 500, 37
    g = gen(C)
    counts = torch.randint(0, 30, (B, M), generator=g, device=dev())
    counts = (counts.double() * ((N - 60) / counts.sum(1, keepdim=True).double())).floor().long()
    counts[:, 3] = 0; counts[:, 4] = 1; counts[0, 9] = 0                # empty and one-row segments
    counts[:, -1] += N - counts.sum(1)                                  # the segments tile all N rows
    off = torch.zeros((B, M + 1), dtype=torch.long, device=dev()); off[:, 1:] = counts.cumsum(1)
    off32 = off.to(i32)
    ldg, ldo = C + 4, C + 12
    G = randn(B * N, ldg, g=g)
    out = torch.full((B * M, ldo), 7.0, device=dev())
    call("usip_seg_sum", P(G), ldg, P(off32), P(out), ldo, B, N, M, C)
    torch.cuda.synchronize()
    Gv = G.view(B, N, ldg)[:, :, :C]
    ref = torch.zeros((B, M, C), device=dev())
    for r in range(int(counts.max())):                                  # row r of every segment, in order
        idx = (off[:, :M] + r).clamp(max=N - 1)
        v = torch.gather(Gv, 1, idx.unsqueeze(2).expand(B, M, C))
        ref = ref + torch.where((r < counts).unsqueeze(2), v, torch.zeros_like(v))
    assert torch.equal(out[:, :C].view(B, M, C), ref) and bool((out[:, C:] == 7.0).all())
    assert bool((out.view(B, M, ldo)[:, 3, :C] == 0).all())


def test_unpool_scatter_bit_exact():
    Pn, Q, C = 3000, 200, 40
    g = gen(5)
    arg = torch.stack([torch.randperm(Pn, generator=g, device=dev())[:Q] for _ in range(C)], 1).to(i32)   # unique per column
    arg[::9] = -1                                                       # empty nodes
    ldp, ldg = C + 7, C + 3
    gp = randn(Q, ldp, g=g)
    for acc in (0, 1):
        G0 = randn(Pn, ldg, g=g)
        G = G0.clone()
        call("usip_unpool_scatter", P(G), ldg, P(gp), ldp, P(arg), Q, C, acc)
        torch.cuda.synchronize()
        ref = G0.clone()
        ok = arg >= 0
        qs, cs = torch.nonzero(ok, as_tuple=True)
        rows = arg[qs, cs].long()
        ref[rows, cs] = (ref[rows, cs] + gp[qs, cs]) if acc else gp[qs, cs]
        assert torch.equal(G, ref), acc


# ================================================================================ kNN combine
@pytest.mark.parametrize("C", [128, 256, 260])
def test_knn_combine_fwd_and_bwd(C):
    B, M, K = 2, 96, 16
    g = gen(C)
    pts = randn(B, 3, M, g=g, scale=3.0)
    knn = torch.randint(0, M, (B, M, K), generator=g, device=dev()).to(i32)
    knn[:, :, 0] = 5                                                    # every node shares neighbour 5: atomics collide
    knn[0, :40, 1:4] = 7
    Q, Gr = B * M, B * M * K
    # forward: Y = Z[nbr] + Wxyz . delta + bias
    ldz, ldw, ldy = C + 4, C + 3 + 5, C + 8
    Z = randn(Q, ldz, g=g)
    W = randn(C, ldw, g=g)
    bias = randn(C, g=g)
    Y = torch.full((Gr, ldy), 7.0, device=dev())
    call("usip_knn_combine", P(Z), ldz, P(pts), P(knn), P(W), ldw, P(bias), P(Y), ldy, None, B, M, K, C)
    torch.cuda.synchronize()
    y_ref = R.knn_combine_fwd(Z[:, :C].double(), pts.double(), knn, W[:, :3].double(), bias.double())
    # three fp32 fmas and two adds per element: measured <= 1.4e-7
    check("knn_combine fwd C=%d" % C, rel(Y[:, :C], y_ref), 1e-6)
    assert bool((Y[:, C:] == 7.0).all())
    # backward, both GZ paths: aligned with ld % 4 == 0 (16-byte atomics) and a column view at offset 1 (scalar atomics)
    ldg = C + 4
    GY = randn(Gr, ldg, g=g)
    GY[:, C:] = NAN
    gz_ref, gw_ref = R.knn_combine_bwd(GY[:, :C].double(), pts.double(), knn, Q)
    for vec in (True, False):
        GZb = torch.zeros((Q, C + (0 if vec else 3)), device=dev())
        GZ, ldzz = (GZb, C) if vec else (GZb[:, 1:], C + 3)
        gWb = randn(C, 3 + 61, g=g)                                     # gW[:, 0:3] of a [C, 3 + C1] weight gradient
        gW0 = gWb.clone()
        call("usip_knn_combine_bwd", P(GY), ldg, P(pts), P(knn), P(GZ), ldzz, P(gWb), gWb.shape[1], B, M, K, C)
        torch.cuda.synchronize()
        tag = "C=%d %s" % (C, "vec" if vec else "scalar")
        # atomics over <= M*K rows per neighbour: measured <= 4.0e-7
        check("knn_combine_bwd GZ " + tag, rel(GZ[:, :C], gz_ref), 2e-6)
        # per-CTA fp32 partials, then atomics: measured <= 2.3e-7
        check("knn_combine_bwd gW " + tag, rel(gWb[:, :3] - gW0[:, :3], gw_ref), 1e-6)
        assert torch.equal(gWb[:, 3:], gW0[:, 3:])
        if not vec:
            assert bool((GZb[:, 0] == 0).all()) and bool((GZb[:, C + 1:] == 0).all())


# ================================================================================ colsum
@pytest.mark.parametrize("C,Pn,slow", [(4, 70000, False), (64, 70000, False), (128, 5000, False), (1024, 3000, False),
                                       (6, 5000, True), (1030, 2100, True)])
def test_colsum(C, Pn, slow):
    g = gen(C + Pn)
    ld = C + (4 if not slow else 3)
    G = randn(Pn, ld, g=g)
    G[-1, :C] = 100.0                                                   # the last row carries weight
    out0 = randn(C, g=g)
    out = out0.clone()
    call("usip_colsum", P(G), ld, P(out), Pn, C)
    torch.cuda.synchronize()
    ref = out0.double() + G[:, :C].double().sum(0)
    mag = out0.double().abs() + G[:, :C].double().abs().sum(0)
    # fp32 partial sums and per-CTA atomics: measured <= 9.0e-8 of sum|term|
    check("colsum C=%d P=%d" % (C, Pn), red(out, ref, mag), 5e-7)


# ================================================================================ head
def test_head_finalize_and_bwd():
    B, M, ld = 3, 100, 7
    g = gen(11)
    out4 = randn(B * M, ld, g=g, scale=4.0)
    out4[0, 3], out4[1, 3], out4[2, 3], out4[3, 3] = 25.0, -50.0, 20.0, 19.5
    out4[4:20, 3] = torch.linspace(0.5, 19.0, 16, device=dev())         # (0, 20]: sigmoid, not the x > 20 shortcut
    out4[20, 3] = float(np.nextafter(np.float32(20), np.float32(21)))   # the first value above the softplus threshold
    out4[21, 3] = -100.0                                                # expf underflows to a subnormal
    cmean = randn(B, 3, M, g=g)
    kp, sig = torch.empty(B, 3, M, device=dev()), torch.empty(B, M, device=dev())
    call("usip_head_finalize", P(out4), ld, P(cmean), 0.001, P(kp), P(sig), B, M)
    g_kp, g_sig = randn(B, 3, M, g=g), randn(B, M, g=g)
    outs = {}
    for name, a, b in (("both", g_kp, g_sig), ("no_kp", None, g_sig), ("no_sig", g_kp, None), ("none", None, None)):
        Gh = torch.full((B * M, 4), NAN, device=dev())
        call("usip_head_bwd", P(a), P(b), P(out4), ld, P(Gh), B, M)
        outs[name] = (Gh, a, b)
    torch.cuda.synchronize()
    kp_ref, sig_ref = R.head_fwd(out4.double()[:, :4].contiguous(), cmean.double(), 0.001)
    assert torch.equal(kp, (out4[:, :3].view(B, M, 3).permute(0, 2, 1) + cmean))      # one fp32 add
    # log1pf(expf(x)): measured <= 3.4e-8
    check("head_finalize sigma", rel(sig, sig_ref), 2e-7)
    x = out4[:, 3].double()
    for name, (Gh, a, b) in outs.items():
        ref = R.head_bwd(None if a is None else a.double(), None if b is None else b.double(), x, B, M)
        assert torch.equal(Gh[:, :3], ref[:, :3].float()), name        # a copy
        err = float((Gh[:, 3].double() - ref[:, 3]).abs().max() / ref[:, 3].abs().max().clamp_min(1e-30)) if b is not None \
            else float(Gh[:, 3].abs().max())
        # 1/(1 + expf(-x)): measured <= 8.5e-8
        check("head_bwd %s" % name, err, 5e-7)


# ================================================================================ wgrad
def _tf32(t):
    """cvt.rna.tf32.f32 on a float32 tensor: round to nearest, ties away from zero, keep 10 mantissa bits."""
    b = t.contiguous().view(i32)
    return ((b + 0x1000) & -0x2000).view(f32)


def _act(X, sc, sh, relu):
    A = X.double()
    if sc is not None:
        A = A * sc.double() + sh.double()
    return A.clamp_min(0) if relu else A


WGRAD_CASES = [
    # name,              P,     Cout, Cin, prec, prologue
    ("tc3x_bn64",        4100,  128,  64,  1,    "affine_relu"),
    ("tc3x_bn128",       5000,  64,   128, 1,    "affine_relu"),
    ("tc3x_relu_only",   4096,  128,  128, 1,    "relu"),
    ("tc3x_none",        4096,  256,  64,  1,    "none"),
    ("simt_cout4",       1000,  4,    256, 1,    "affine_relu"),
    ("simt_cout6",       3000,  6,    131, 1,    "affine_relu"),
    ("simt_cin131",      5000,  130,  131, 1,    "relu"),
    ("simt_small_p",     3000,  128,  128, 1,    "none"),
    ("simt_prec0",       6000,  64,   64,  0,    "affine_relu"),
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=[c[0] for c in WGRAD_CASES])
def test_wgrad_paths(case):
    """3xTF32 wgmma at BN 64 / 128, the fp32 SIMT kernel (narrow Cout, Cout % 4 != 0, Cin = 131, P < 4096), with and
    without the BN prologue and ReLU; X a column view of a wider buffer, gW a column slice accumulated into."""
    name, Pn, Cout, Cin, prec, pro = case
    g = gen(Pn + Cout + Cin)
    ldx = Cin + 64 + (Cin % 4 and 1)                                    # X = AGG[:, :Cin]
    AGG = randn(Pn, ldx, g=g)
    GY = randn(Pn, Cout, g=g)
    sc = randn(Cin, g=g) if pro == "affine_relu" else None
    sh = randn(Cin, g=g) if pro == "affine_relu" else None
    relu = pro != "none"
    ref = R.wgrad(GY.double(), _act(AGG[:, :Cin], sc, sh, False), None, None, relu)
    for off in (3, 64):                                                 # gW[:, 3:] (odd column: scalar epilogue), gW[:, Cb:]
        gWb = randn(Cout, off + Cin, g=g)
        gW0 = gWb.clone()
        call("usip_wgrad", P(GY), Cout, P(AGG), ldx, P(sc), P(sh), 1 if relu else 0, P(gWb, off), off + Cin, Pn, Cout, Cin, prec)
        torch.cuda.synchronize()
        # split-K fp32 partials and atomics: measured <= 1.2e-6 on the 3xTF32 kernel, <= 3.9e-7 on the SIMT kernel
        check("wgrad %s off=%d" % (name, off), rel(gWb[:, off:] - gW0[:, off:], ref), 5e-6 if name.startswith("tc") else 2e-6)
        assert torch.equal(gWb[:, :off], gW0[:, :off])


def test_wgrad_plain_tf32():
    """precision 4: single-pass TF32 on the same wgmma kernel, against a reference on TF32-rounded operands."""
    Pn, Cout, Cin = 4096, 128, 128
    g = gen(44)
    X, GY = randn(Pn, Cin, g=g), randn(Pn, Cout, g=g)
    sc, sh = randn(Cin, g=g), randn(Cin, g=g)
    gW = torch.zeros((Cout, Cin), device=dev())
    call("usip_wgrad", P(GY), Cout, P(X), Cin, P(sc), P(sh), 1, P(gW), Cin, Pn, Cout, Cin, 4)
    torch.cuda.synchronize()
    A = torch.clamp_min(torch.addcmul(sh, X, sc), 0)                   # fp32 fma like the kernel's prologue
    ref = _tf32(GY).double().t() @ _tf32(A).double()
    # fp32 accumulation of TF32 products: measured <= 3.6e-7 against the TF32-rounded reference
    check("wgrad tf32", rel(gW, ref), 2e-6)
    exact = GY.double().t() @ A.double()
    assert rel(gW, exact) > 5e-6                                        # it really is single-pass TF32


@pytest.mark.parametrize("Cout", [32, 64, 128, 256])
def test_wgrad_narrow(Cout):
    """The first layer (Cin <= 8): the row-streaming kernel with the packed 8-column X (ldx == 8, NaN in the padding
    columns) and with a generic ldx."""
    Pn = 5000
    for Cin in (3, 7, 8):
        for ldx in (8, 11):
            g = gen(Cout * 100 + Cin * 10 + ldx)
            X = torch.full((Pn, ldx), NAN, device=dev()); X[:, :Cin] = randn(Pn, Cin, g=g)
            GY = randn(Pn, Cout, g=g)
            sc, sh = randn(Cin, g=g), randn(Cin, g=g)
            for relu in (1, 0):
                gW = randn(Cout, Cin, g=g)
                gW0 = gW.clone()
                call("usip_wgrad", P(GY), Cout, P(X), ldx, P(sc), P(sh), relu, P(gW), Cin, Pn, Cout, Cin, 1)
                torch.cuda.synchronize()
                ref = R.wgrad(GY.double(), X[:, :Cin].double(), sc.double(), sh.double(), bool(relu))
                # per-thread fp32 chains over P / (2 SMs * rows per pass) rows: measured <= 4.4e-7
                check("wgrad narrow Cout=%d Cin=%d ldx=%d relu=%d" % (Cout, Cin, ldx, relu), rel(gW - gW0, ref), 2e-6)


# ================================================================================ descriptor head
def test_l2norm_fwd_and_bwd():
    B, M, C = 2, 50, 100                                                # C not a multiple of 32
    g = gen(12)
    ldx, ldo = C + 7, C + 3
    X = randn(B * M, ldx, g=g)
    X[5, :C] = 0.0                                                      # zero norm
    X[6:12, :C] *= 3e-6                                                 # norms near the 1e-5 epsilon
    out = torch.empty(B, C, M, device=dev()); nrm = torch.empty(B * M, device=dev())
    call("usip_l2norm_to_bcm", P(X), ldx, P(out), P(nrm), B, M, C)
    gg = randn(B, C, M, g=g)
    GY = torch.full((B * M, ldo), 7.0, device=dev())
    call("usip_l2norm_bwd", P(gg), P(X), ldx, P(GY), ldo, B, M, C)
    torch.cuda.synchronize()
    Xd = X[:, :C].double()
    # fp32 warp-shuffle norms: measured <= 1.3e-7
    check("l2norm fwd", rel(out, R.l2norm_fwd(Xd, B, M)), 1e-6)
    check("l2norm norm", rel(nrm, Xd.norm(dim=1)), 5e-7)
    ref = R.l2norm_bwd(gg.double(), Xd, B, M)
    # measured <= 4.4e-8; the zero and near-epsilon rows dominate max|ref|, so the O(1) rows are checked on their own too
    check("l2norm bwd", rel(GY[:, :C], ref), 5e-7)
    big = ref.abs().amax(1) > 0
    rows = torch.arange(B * M, device=dev())
    ok = (rows < 6) | (rows >= 12)
    check("l2norm bwd O(1) rows", rel(GY[:, :C][ok & big], ref[ok & big]), 5e-7)
    assert bool((GY[:, C:] == 7.0).all())


def test_desc_triplet_fwd_and_bwd():
    B, C, M, Mp, Mn = 2, 32, 200, 150, 90
    gamma, smax = 0.5, 3.0
    g = gen(13)
    anc, pos, neg = randn(B, C, M, g=g), randn(B, C, Mp, g=g), randn(B, C, Mn, g=g)
    ipos = torch.randint(0, Mp, (B, M), generator=g, device=dev()).to(i32)
    ineg = torch.randint(0, Mn, (B, M), generator=g, device=dev()).to(i32)
    ipos[:, :10] = 2; ineg[:, 5:15] = 4                                  # several anchors share one match
    pos[0, :, 3] = anc[0, :, 1]; ipos[0, 1] = 3                          # dpos = 0
    neg[1, :, 0] = anc[1, :, 2]; ineg[1, 2] = 0                          # dneg = 0
    sigma = rand(B, M, g=g) * 2.5
    sigma[0, 7] = 3.0; sigma[1, 8] = 4.0                                 # sigma >= sigma_max: weight 0
    dpos = (anc.double() - R._col_gather(pos.double(), ipos)).norm(dim=1)
    dneg = (anc.double() - R._col_gather(neg.double(), ineg)).norm(dim=1)
    h = dpos - dneg + gamma
    sigma = torch.where(h.abs() < 1e-3, torch.full_like(sigma, 3.5), sigma)    # an undecided hinge gets weight 0
    dp32, dn32 = dpos.float(), dneg.float()
    assert bool((h > 0).any()) and bool((h < 0).any())
    loss, active = torch.empty(B, M, device=dev()), torch.empty(B, device=dev())
    call("usip_desc_triplet", P(dp32), P(dn32), P(sigma), gamma, smax, P(loss), P(active), B, M)
    g_loss = randn(B, M, g=g)
    ga, gp, gn = torch.zeros_like(anc), torch.zeros_like(pos), torch.zeros_like(neg)
    call("usip_desc_triplet_bwd", P(anc), P(pos), P(neg), P(dp32), P(ipos), P(dn32), P(ineg), P(sigma), gamma, smax,
         P(g_loss), P(ga), P(gp), P(gn), B, C, M, Mp, Mn)
    torch.cuda.synchronize()
    l_ref, a_ref = R.desc_triplet_fwd(dp32.double(), dn32.double(), sigma.double(), gamma, smax)
    # measured <= 4.2e-8
    check("desc_triplet loss", rel(loss, l_ref), 5e-7)
    assert torch.equal(active, a_ref.float())
    refs = R.desc_triplet_bwd(anc.double(), pos.double(), neg.double(), ipos, ineg, sigma.double(), gamma, smax, g_loss.double())
    for nm, got, ref in (("anc", ga, refs[0]), ("pos", gp, refs[1]), ("neg", gn, refs[2])):
        # fp32 per-term arithmetic, atomics over shared matches: measured <= 2.0e-7
        check("desc_triplet_bwd " + nm, rel(got, ref), 1e-6)
    assert float(ga[0, :, 7].abs().max()) == 0 and float(ga[1, :, 8].abs().max()) == 0


# ================================================================================ detector losses
def test_transform_points_fwd_and_bwd():
    B, M = 4, 300
    g = gen(14)
    kp, Rm = randn(B, 3, M, g=g, scale=10.0), randn(B, 3, 3, g=g)
    sc, sh = rand(B, g=g) + 0.5, randn(B, 3, g=g)
    out = torch.empty_like(kp)
    call("usip_transform_points", P(kp), P(Rm), P(sc), P(sh), P(out), B, M)
    gout = randn(B, 3, M, g=g)
    gk = torch.full_like(kp, NAN)
    call("usip_transform_points_bwd", P(gout), P(Rm), P(sc), P(gk), B, M)
    torch.cuda.synchronize()
    # measured <= 8.4e-8
    check("transform_points", rel(out, R.transform_points_fwd(kp.double(), Rm.double(), sc.double(), sh.double())), 5e-7)
    check("transform_points_bwd", rel(gk, R.transform_points_bwd(gout.double(), Rm.double(), sc.double())), 5e-7)


def test_pairwise_min_bwd():
    B, Ma, Nb = 2, 300, 120
    g = gen(15)
    a, b = randn(B, 3, Ma, g=g), randn(B, 3, Nb, g=g)
    arg = torch.randint(0, Nb, (B, Ma), generator=g, device=dev()).to(i32)
    arg[:, :20] = 4                                                     # repeated j
    a[0, :, 30] = b[0, :, int(arg[0, 30])]                              # d = 0
    d = (a.double() - R._col_gather(b.double(), arg)).norm(dim=1).float()
    gv = randn(B, Ma, g=g)
    for gname, gg in (("g", gv), ("null g", None)):
        ga_ref, gb_ref = R.pairwise_min_bwd(a.double(), b.double(), d.double(), arg, None if gg is None else gg.double(), 0.37)
        ga, gb = torch.full_like(a, NAN), torch.zeros_like(b)
        call("usip_pairwise_min_bwd", P(a), P(b), P(d), P(arg), P(gg), 0.37, P(ga), P(gb), B, Ma, Nb)
        ga2 = torch.full_like(a, NAN)
        call("usip_pairwise_min_bwd", P(a), P(b), P(d), P(arg), P(gg), 0.37, P(ga2), None, B, Ma, Nb)
        gb2 = torch.zeros_like(b)
        call("usip_pairwise_min_bwd", P(a), P(b), P(d), P(arg), P(gg), 0.37, None, P(gb2), B, Ma, Nb)
        torch.cuda.synchronize()
        # measured <= 1.2e-7 (grad_b: atomics over the repeated j)
        check("pairwise_min_bwd ga " + gname, rel(ga, ga_ref), 5e-7)
        check("pairwise_min_bwd gb " + gname, rel(gb, gb_ref), 5e-7)
        assert torch.equal(ga2, ga)
        check("pairwise_min_bwd gb only " + gname, rel(gb2, gb_ref), 5e-7)
        assert float(ga[0, :, 30].abs().max()) == 0


def test_chamfer_prob_reduce_and_bwd():
    B, M, N = 2, 256, 320
    g = gen(16)
    src, dst = randn(B, 3, M, g=g), randn(B, 3, N, g=g)
    i_sd = torch.randint(0, N, (B, M), generator=g, device=dev()).to(i32)
    i_ds = torch.randint(0, M, (B, N), generator=g, device=dev()).to(i32)
    src[1, :, 2] = dst[1, :, int(i_sd[1, 2])]                           # d = 0
    ss, sd = rand(B, M, g=g) + 0.2, rand(B, N, g=g) + 0.2
    d_sd = (src.double() - R._col_gather(dst.double(), i_sd)).norm(dim=1).float()
    d_ds = (dst.double() - R._col_gather(src.double(), i_ds)).norm(dim=1).float()
    out3 = torch.empty(3, device=dev())
    call("usip_chamfer_prob_reduce", P(d_sd), P(i_sd), P(d_ds), P(i_ds), P(ss), P(sd), P(out3), B, M, N)
    gout = torch.tensor([1.7], device=dev())
    grads = [torch.zeros_like(t) for t in (src, dst, ss, sd)]
    call("usip_chamfer_prob_bwd", P(src), P(dst), P(ss), P(sd), P(d_sd), P(i_sd), P(d_ds), P(i_ds), P(gout), *[P(t) for t in grads],
         B, M, N)
    torch.cuda.synchronize()
    ref = R.chamfer_prob_fwd(src.double(), dst.double(), ss.double(), sd.double(), i_sd, i_ds)
    # fp32 per-element terms, float64 sums: measured <= 2.2e-8
    check("chamfer_prob_reduce", rel(out3, torch.stack(list(ref))), 2e-7)
    refs = R.chamfer_prob_bwd(src.double(), dst.double(), ss.double(), sd.double(), i_sd, i_ds, 1.7)
    for nm, got, r in zip(("src", "dst", "sig_src", "sig_dst"), grads, refs):
        # atomics of fp32 terms: measured <= 1.4e-7
        check("chamfer_prob_bwd " + nm, rel(got, r), 1e-6)


def test_point_on_surface_with_grad():
    B, M, N, S = 2, 200, 500, 4
    g = gen(17)
    kp, pc, sn = randn(B, 3, M, g=g), randn(B, 3, N, g=g), randn(B, S, N, g=g)
    arg = torch.randint(0, N, (B, M), generator=g, device=dev()).to(i32)
    kp[0, :, 1] = pc[0, :, int(arg[0, 1])]                              # r = 0
    gv = randn(B, M, g=g)
    loss, gk = torch.empty(B, M, device=dev()), torch.empty(B, 3, M, device=dev())
    call("usip_point_on_surface", P(kp), P(pc), P(sn), P(arg), P(gv), P(loss), P(gk), B, M, N, S)
    torch.cuda.synchronize()
    l_ref, g_ref = R.point_on_surface(kp.double(), pc.double(), sn.double(), arg, gv.double())
    # measured <= 1.7e-7
    check("point_on_surface loss", rel(loss, l_ref), 5e-7)
    check("point_on_surface g_kp", rel(gk, g_ref), 1e-6)


# ================================================================================ misaligned operands
def test_backward_entry_points_reject_misaligned_device_operands():
    """Each guarded entry point called with one real device operand one float off a 16-byte boundary raises
    RuntimeError before any launch (usip_b200.h, section 5)."""
    C, Pn, K, Q = 64, 256, 16, 16
    buf = lambda *s: torch.zeros(*s, device=dev())
    G, Y, GY, part = buf(Pn, C + 4), buf(Pn, C + 4), buf(Pn, C + 4), buf(2, 2, C + 4)
    v = [buf(C + 4) for _ in range(6)]
    gz, argsel = buf(Q, C + 4), torch.zeros(Q, C + 4, dtype=i32, device=dev())
    seg = torch.zeros(1, 2, dtype=i32, device=dev())
    pts, knn = buf(1, 3, Q), torch.zeros(1, Q, K, dtype=i32, device=dev())
    cases = [
        ("usip_bn_bwd_reduce", lambda o: (P(G, o), C, P(Y), C, P(v[0]), P(v[1]), P(v[2]), P(v[3]), 1, P(part), Pn, C)),
        ("usip_bn_bwd_reduce", lambda o: (P(G), C, P(Y), C, P(v[0], o), P(v[1]), P(v[2]), P(v[3]), 1, P(part), Pn, C)),
        ("usip_bn_bwd_apply", lambda o: (P(G), C, P(Y), C, P(v[0]), P(v[1]), P(v[2]), P(v[3]), P(v[4]), P(v[5]), 1, P(GY, o), C, Pn, C)),
        ("usip_bn_bwd_apply", lambda o: (P(G), C, P(Y, o), C, P(v[0]), P(v[1]), P(v[2]), P(v[3]), P(v[4]), P(v[5], o), 1, P(GY), C, Pn, C)),
        ("usip_groupmax_bwd_apply", lambda o: (P(Y), C, P(gz, o), P(argsel), P(v[0]), P(v[1]), P(v[2]), P(v[3]), P(v[4]), P(GY), C, K, Pn, C)),
        ("usip_groupmax_bwd_apply", lambda o: (P(Y), C, P(gz), P(argsel, o), P(v[0]), P(v[1]), P(v[2]), P(v[3]), P(v[4]), P(GY), C, K, Pn, C)),
        ("usip_group_sum", lambda o: (P(G, o), C, P(gz), C, K, Q, C)),
        ("usip_group_sum", lambda o: (P(G), C, P(gz, o), C, K, Q, C)),
        ("usip_seg_sum", lambda o: (P(G, o), C, P(seg), P(gz), C, 1, Pn, 1, C)),
        ("usip_head_bwd", lambda o: (None, None, P(G), 4, P(GY, o), 1, Q)),
        ("usip_knn_combine_bwd", lambda o: (P(GY, o), C, P(pts), P(knn), P(gz), C, P(part), 3, 1, Q, K, C)),
    ]
    for name, args in cases:
        call(name, *args(0))                                            # aligned: accepted
        with pytest.raises(RuntimeError, match="aligned"):
            call(name, *args(1))
    torch.cuda.synchronize()


# ================================================================================ Adam
def test_flat_adam_matches_torch_adam_and_counts_steps():
    """FlatAdam / usip_adam_step: five steps with different gradients, an lr change and grad_scale != 1 on parameters
    whose sizes need padding, against torch.optim.Adam in float64; step_dev advances by one per launch, also when one
    captured step is replayed as a CUDA graph."""
    from usip_b200.optim import FlatAdam
    g = gen(18)
    shapes = [(5,), (3, 7), (13,), (64, 3), (1,)]
    # parameters of the size of a few updates, so the fp32 storage of p does not hide the error of the update itself
    params = [torch.nn.Parameter(randn(*s, g=g, scale=1e-3)) for s in shapes]
    init = [p.detach().clone() for p in params]
    opt = FlatAdam(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    opt.grad_scale = 0.5
    lrs = [1e-3, 1e-3, 3e-3, 3e-3, 5e-4]
    grads = [[randn(*s, g=g) * (1 + t) for s in shapes] for t in range(5)]
    for t in range(5):
        opt.param_groups[0]["lr"] = lrs[t]
        for p, gr in zip(params, grads[t]):
            p.grad.copy_(gr)
        opt.step()
        assert int(opt.step_dev.item()) == t + 1
    torch.cuda.synchronize()
    # the C ABI takes the betas as float: the reference runs with those fp32 values (with the float64 0.999, torch's
    # exp_avg_sq is 1.3e-5 larger -- 1 - 0.999f is 1.3e-5 below 0.001 -- while the bias correction, which uses the same
    # beta, cancels it in the update)
    betas = (float(np.float32(0.9)), float(np.float32(0.999)))
    p_ref, m_ref, v_ref = R.adam_reference(init, grads, lrs, betas, 1e-8, 0.5)
    path = sum(lrs)                                                     # an Adam step moves a parameter by about lr
    for i, p in enumerate(params):
        # parameters, relative to the summed step sizes: measured <= 1.4e-7 (also against float64 betas); moments: <= 8.8e-8
        check("adam p[%d]" % i, float((p.detach().double() - p_ref[i]).abs().max()) / path, 1e-6)
        check("adam exp_avg[%d]" % i, rel(opt.state[p]["exp_avg"], m_ref[i]), 1e-6)
        check("adam exp_avg_sq[%d]" % i, rel(opt.state[p]["exp_avg_sq"], v_ref[i]), 1e-6)
    p_t, _, _ = R.adam_reference(init, grads, lrs, (0.9, 0.999), 1e-8, 0.5)
    for i, p in enumerate(params):
        check("adam p[%d] vs float64 betas" % i, float((p.detach().double() - p_t[i]).abs().max()) / path, 1e-6)
    # one captured step, replayed three times with the same gradient
    gfix = [randn(*s, g=g) for s in shapes]
    for p, gr in zip(params, gfix):
        p.grad.copy_(gr)
    before = [p.detach().clone() for p in params]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            opt.step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert int(opt.step_dev.item()) == 5                                # capturing does not run the step
    assert all(torch.equal(p.detach(), b) for p, b in zip(params, before))
    for r in range(3):
        graph.replay()
        torch.cuda.synchronize()
        assert int(opt.step_dev.item()) == 6 + r
    p_ref, _, _ = R.adam_reference(init, grads + [gfix] * 3, lrs + [5e-4] * 3, betas, 1e-8, 0.5)
    for i, p in enumerate(params):
        check("adam graph p[%d]" % i, float((p.detach().double() - p_ref[i]).abs().max()) / (path + 3 * 5e-4), 1e-6)
    with pytest.raises(RuntimeError):
        call("usip_adam_step", P(opt.flat_p), P(opt.flat_g), P(opt.exp_avg), P(opt.exp_avg_sq), P(opt.lr_dev),
             P(opt.step_dev), P(opt._arrive), 0.9, 0.999, 1e-8, 1.0, opt.n - 1)   # n % 4 != 0
