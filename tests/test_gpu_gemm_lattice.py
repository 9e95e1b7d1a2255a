"""-m gpu: the layer GEMM (usip_layer_fwd: row-warp, narrow, SIMT<64> / SIMT<128> and wgmma kernels) and the weight-gradient
GEMM (usip_wgrad: narrow, SIMT and wgmma kernels) on dyadic lattices (tests/gemm_ref.py), where every path must equal its
float64 restatement BIT FOR BIT: Y, the BN-statistic partial of every slot, the group max / min and their rows (ties go
to the first row of the group), gW after +=.  On the lo lattices fp32 and 3xTF32 give the exact product and plain TF32
gives sum hi*hi, a different value, so the output also says which path ran and whether the compensation terms are there.
Every case asserts, from the dispatch restatement and the device's SM count, that it reaches the kernel it was written
for.  Memory a call must not read holds NaN (padding columns, rows past P, columns 3..7 of the narrow kernel's vector
load, W columns past Cin); memory it must not write holds a sentinel that must survive.

Off the lattice: each element of the 3xTF32 layer and wgrad output stays within tau * sum_k |a_k| |w_k| (+ |bias|) of the
float64 product, and plain TF32 on the same inputs is at least 64x worse.  Each bound prints the worst error measured
beside it; gemm_ref.TAU_LAYER / TAU_WGRAD give the values measured on an H100 80GB HBM3 (SXM, 700 W power limit).
The layer kernels are deterministic: two launches give the same bits."""
import ctypes

import numpy as np
import pytest
import torch

from tests import gemm_ref as G

pytestmark = pytest.mark.gpu

NAN = float("nan")
SENT = -7777.25                       # sentinel in memory a call must not write


def _lib():
    from usip_b200 import _lib as L
    return L


def _stream():
    from usip_b200.ops import _stream as s
    return s()


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cu(a, dtype=torch.float32):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def addr(t):
    return None if t is None else t.data_ptr()


class Buf:
    """A [rows, cols] operand with row stride ld, `off` floats into an allocation filled with `fill` (NaN: must not be
    read; SENT: must not be written) that also holds `extra` rows past the last one."""

    def __init__(self, vals, ld, off=0, fill=NAN, extra=2):
        vals = np.asarray(vals, np.float32)
        self.rows, self.cols = vals.shape
        self.ld, self.off, self.fill = ld, off, fill
        self.t = torch.full((off + (self.rows + extra) * ld,), fill, device="cuda")
        self.view().copy_(cu(vals))

    def view(self):
        return self.t[self.off:self.off + self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols]

    def ptr(self):
        return self.t.data_ptr() + 4 * self.off

    def untouched(self):
        m = torch.ones_like(self.t, dtype=torch.bool)
        m[self.off:self.off + self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols] = False
        out = self.t[m]
        return bool(torch.isnan(out).all()) if self.fill != self.fill else bool((out == self.fill).all())


def exact(what, got, ref):
    """got (device) == ref (float64 on the fp32 lattice), element for element."""
    g = got.cpu().numpy().astype(np.float64) if torch.is_tensor(got) else np.asarray(got, np.float64)
    bad = g != ref
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r want %r"
                             % (what, int(bad.sum()), bad.size, tuple(i), g[tuple(i)], ref[tuple(i)]))


def _mode(path):
    return "tf32" if "+tf32" in path else ("3x" if path.startswith("tc") else "fp32")


# ============================================================================ usip_layer_fwd on the lattices
def _layer_desc(P, Cin, Cout, X, W, wt, op, Y, prec, part=None, grp=None, ws=None, packed=False):
    d = _lib().LayerDesc()
    d.X = X.ptr(); d.ldx = X.ld; d.P = P; d.Cin = Cin; d.Cout = Cout
    d.W = W.ptr(); d.ldw = W.ld; d.w_transposed = 1 if wt else 0
    d.bias = addr(op["_bias"]); d.in_scale = addr(op["_scale"]); d.in_shift = addr(op["_shift"]); d.in_relu = int(op["relu"])
    if op["_add"] is not None:
        d.addend = addr(op["_add"]); d.ld_add = Cout
        d.add_index = addr(op["_add_index"]); d.add_group = op["add_group"] or 0
    d.Y = Y.ptr(); d.ldy = Y.ld
    d.stat_partial = addr(part)
    if grp:
        d.gmax, d.gmin = addr(grp["gmax"]), addr(grp["gmin"])
        d.garg_max, d.garg_min = addr(grp.get("amax")), addr(grp.get("amin"))
        d.group = grp["g"]
    if prec != "fp32":
        d.precision = 1
        d.debug_flags = 8 if prec == "tf32" else 0
        d.tc_workspace = ws.data_ptr(); d.tc_workspace_bytes = ws.numel() * 4; d.tc_weights_packed = int(packed)
    return d


def _upload(op):
    op["_bias"], op["_scale"], op["_shift"] = cu(op["bias"]), cu(op["scale"]), cu(op["shift"])
    op["_add"], op["_add_index"] = cu(op["addend"]), cu(op["add_index"], torch.int32)
    return op


def run_layer(cid, P, Cin, Cout, kw, with_args=True):
    sm = sm_count()
    prec, group, stats = kw["prec"], kw.get("group", 0), bool(kw.get("stats"))
    path = G.layer_path(P, Cin, Cout, sm, precision=0 if prec == "fp32" else 1, single=prec == "tf32", stats=stats,
                        group=group, addend=bool(kw.get("add")), affine=kw["pro"].startswith("affine"),
                        relu=kw["pro"] in ("affine_relu", "relu"))
    assert path == kw["path"], (cid, path, "the case no longer reaches the kernel it was written for")
    op = _upload(G.layer_operands(G.case_seed(cid), P, Cin, Cout, kw["kind"], kw["pro"], kw.get("add"),
                                  wdens=kw.get("wdens", 1.0), ties=kw.get("ties", 0)))
    wt = bool(kw.get("wt"))
    Wm = np.ascontiguousarray(op["W"].T) if wt else op["W"]
    X = Buf(op["X"], Cin + kw.get("ldx_pad", 0), kw.get("x_off", 0))
    W = Buf(Wm, Wm.shape[1] + kw.get("ldw_pad", 0), kw.get("w_off", 0))
    Y = Buf(np.full((P, Cout), SENT, np.float32), Cout + kw.get("ldy_pad", 0), fill=SENT)
    grp = None
    if group:
        Q = P // group
        grp = dict(g=group, gmax=torch.full((Q, Cout), SENT, device="cuda"), gmin=torch.full((Q, Cout), SENT, device="cuda"))
        if with_args:
            grp["amax"] = torch.full((Q, Cout), -1, dtype=torch.int32, device="cuda")
            grp["amin"] = torch.full((Q, Cout), -1, dtype=torch.int32, device="cuda")
    ws = torch.empty(2 * Cin * Cout, device="cuda") if prec != "fp32" else None
    part = None
    if stats:
        probe = _layer_desc(P, Cin, Cout, X, W, wt, op, Y, prec, grp=grp, ws=ws)
        probe.stat_partial = 1                                          # the query tests it for NULL only
        nslots = _lib().load().usip_layer_stat_slots(ctypes.byref(probe))
        slots = G.stat_slot_rows(path, P, Cout, sm)
        assert nslots == len(slots), (nslots, len(slots))
        part = torch.full((nslots, 2, Cout), NAN, device="cuda")
    d = _layer_desc(P, Cin, Cout, X, W, wt, op, Y, prec, part=part, grp=grp, ws=ws)
    _lib().check(_lib().load().usip_layer_fwd(ctypes.byref(d), _stream()), "usip_layer_fwd")
    torch.cuda.synchronize()

    ref = G.layer_expect(op, _mode(path))
    exact("%s Y" % cid, Y.view(), ref)
    assert Y.untouched(), "%s: Y written outside [P, Cout]" % cid
    if stats:
        assert G.stats_exact(ref, op["step"], slots)
        exact("%s statistics" % cid, part, G.stats_ref(ref, slots))
    if group:
        mx, mn, amx, amn = G.group_ref(ref, group)
        exact("%s gmax" % cid, grp["gmax"], mx)
        exact("%s gmin" % cid, grp["gmin"], mn)
        if with_args:
            exact("%s garg_max" % cid, grp["amax"], amx)
            exact("%s garg_min" % cid, grp["amin"], amn)
    return Y.view().clone(), grp


@pytest.mark.parametrize("case", G.LAYER_CASES, ids=[c[0] for c in G.LAYER_CASES])
def test_layer_lattice(case):
    cid, P, Cin, Cout, kw = case
    _, g1 = run_layer(cid, P, Cin, Cout, kw, with_args=True)
    if kw.get("group"):
        # without arg outputs (the tensor-core kernel's fmaxf / fminf fast path): the same max / min bits
        _, g0 = run_layer(cid, P, Cin, Cout, kw, with_args=False)
        assert torch.equal(g0["gmax"].view(torch.int32), g1["gmax"].view(torch.int32))
        assert torch.equal(g0["gmin"].view(torch.int32), g1["gmin"].view(torch.int32))


PACK_CASES = [(4100, 64, 128, False, "tc64"), (17000, 256, 256, False, "tc128"), (17000, 256, 128, True, "tc128"),
              (4100, 96, 64, True, "tc64")]


def test_layer_tc_pack_many_matches_inline_pack():
    """usip_layer_tc_pack_many over four layers in ONE launch (both widths, transposed W), then each layer with
    tc_weights_packed = 1: the same workspace bits and the same Y as the inline pack, and Y exact on the lo-W lattice."""
    sm = sm_count()
    descs, keep = [], []
    for i, (P, Cin, Cout, wt, path) in enumerate(PACK_CASES):
        assert G.layer_path(P, Cin, Cout, sm, precision=1) == path
        op = _upload(G.layer_operands(100 + i, P, Cin, Cout, "lo_w", "affine_relu"))
        Wm = np.ascontiguousarray(op["W"].T) if wt else op["W"]
        X, W = Buf(op["X"], Cin), Buf(Wm, Wm.shape[1] + 4)
        Y = Buf(np.full((P, Cout), SENT, np.float32), Cout, fill=SENT)
        ws = torch.full((2 * Cin * Cout,), NAN, device="cuda")
        descs.append(_layer_desc(P, Cin, Cout, X, W, wt, op, Y, "3x", ws=ws, packed=True))
        keep.append((op, X, W, Y, ws, wt))
    arr = (_lib().LayerDesc * len(descs))(*descs)
    _lib().check(_lib().load().usip_layer_tc_pack_many(arr, len(descs), _stream()), "usip_layer_tc_pack_many")
    for d in descs:
        _lib().check(_lib().load().usip_layer_fwd(ctypes.byref(d), _stream()), "usip_layer_fwd")
    for (P, Cin, Cout, wt, path), d, (op, X, W, Y, ws, _) in zip(PACK_CASES, descs, keep):
        Y2 = Buf(np.full((P, Cout), SENT, np.float32), Cout, fill=SENT)
        ws2 = torch.full_like(ws, NAN)
        d2 = _layer_desc(P, Cin, Cout, X, W, wt, op, Y2, "3x", ws=ws2, packed=False)
        _lib().check(_lib().load().usip_layer_fwd(ctypes.byref(d2), _stream()), "usip_layer_fwd")
        torch.cuda.synchronize()
        assert torch.equal(ws.view(torch.int32), ws2.view(torch.int32)), (P, Cin, Cout, wt)
        assert torch.equal(Y.view(), Y2.view())
        exact("packed %s wt=%d" % (path, wt), Y.view(), G.layer_expect(op, "3x"))


# ============================================================================ usip_wgrad on the lattices
@pytest.mark.parametrize("case", G.WGRAD_CASES, ids=[c[0] for c in G.WGRAD_CASES])
def test_wgrad_lattice(case):
    cid, P, Cout, Cin, kw = case
    sm = sm_count()
    P = G.wgrad_case_P(P, Cout, Cin, kw, sm)
    ldg, ldx = Cout + kw.get("ldg_pad", 0), Cin + kw.get("ldx_pad", 0)
    gy_off, x_off = kw.get("gy_off", 0), kw.get("x_off", 0)
    path = G.wgrad_path(P, Cout, Cin, kw["prec"], ldg, ldx, gy_off % 4 == 0, x_off % 4 == 0)
    assert path == kw["path"], (cid, path, "the case no longer reaches the kernel it was written for")
    op = G.wgrad_operands(G.case_seed(cid), P, Cout, Cin, kw["kind"], kw["pro"])
    GY, X = Buf(op["GY"], ldg, gy_off), Buf(op["X"], ldx, x_off)
    gW = Buf(op["gW0"], Cin + kw.get("ldw_pad", 0), fill=SENT)
    sc, sh = cu(op["scale"]), cu(op["shift"])
    _lib().check(_lib().load().usip_wgrad(GY.ptr(), ldg, X.ptr(), ldx, addr(sc), addr(sh), int(op["relu"]), gW.ptr(),
                                          gW.ld, P, Cout, Cin, kw["prec"], _stream()), "usip_wgrad")
    torch.cuda.synchronize()
    exact("%s gW" % cid, gW.view(), G.wgrad_expect(op, _mode(path)))
    assert gW.untouched(), "%s: gW written outside [Cout, Cin]" % cid


# ============================================================================ 3xTF32 error bound off the lattice
def _check_bound(what, got_3x, got_tf32, ref, mag, tau):
    e3 = float((np.abs(got_3x - ref) / mag).max())
    et = float((np.abs(got_tf32 - ref) / mag).max())
    print("measured %-40s 3xTF32 %.3e (tau %.1e)   plain TF32 %.3e  ratio %.0f" % (what, e3, tau, et, et / max(e3, 1e-30)))
    assert e3 <= tau, (what, e3, tau)
    assert et >= 64 * e3, (what, et, e3)


@pytest.mark.parametrize("P,Cin,Cout,path", [(4096, 256, 128, "tc64"), (17000, 256, 128, "tc128")])
def test_layer_3xtf32_error_bound(P, Cin, Cout, path):
    """Operands of gemm_ref.bound_layer_operands: scales spanning 2^+-20 over rows and columns and 2^+-8 over K chunks."""
    assert G.layer_path(P, Cin, Cout, sm_count(), precision=1) == path
    X, Wm, b = G.bound_layer_operands(P, Cin, Cout)
    op = _upload(dict(bias=b, scale=None, shift=None, relu=False, addend=None, add_index=None, add_group=None))
    Xb, Wb = Buf(X, Cin), Buf(Wm, Cin)
    out = {}
    for prec in ("3x", "tf32"):
        Y = Buf(np.zeros((P, Cout), np.float32), Cout, fill=SENT)
        d = _layer_desc(P, Cin, Cout, Xb, Wb, False, op, Y, prec, ws=torch.empty(2 * Cin * Cout, device="cuda"))
        _lib().check(_lib().load().usip_layer_fwd(ctypes.byref(d), _stream()), "usip_layer_fwd")
        torch.cuda.synchronize()
        out[prec] = Y.view().cpu().numpy().astype(np.float64)
    ref = G.layer_ref(X, Wm, b)
    mag = G.err_bound(X, Wm, 1.0, (np.broadcast_to(b, (P, Cout)),))
    _check_bound("layer %s P=%d" % (path, P), out["3x"], out["tf32"], ref, mag, G.TAU_LAYER)


@pytest.mark.parametrize("P,Cout,Cin,path", [(4096, 128, 128, "tc128"), (8203, 100, 192, "tc64")])
def test_wgrad_3xtf32_error_bound(P, Cout, Cin, path):
    """Operands of gemm_ref.bound_wgrad_operands: scales spanning 2^+-20 over output rows and columns and 2^+-10 over 32-row
    chunks of the reduction."""
    assert G.wgrad_path(P, Cout, Cin, 1) == path
    GY, X = G.bound_wgrad_operands(P, Cout, Cin)
    GYb, Xb = Buf(GY, Cout), Buf(X, Cin)
    out = {}
    for prec in (1, 4):
        gW = torch.zeros((Cout, Cin), device="cuda")
        _lib().check(_lib().load().usip_wgrad(GYb.ptr(), Cout, Xb.ptr(), Cin, None, None, 0, gW.data_ptr(), Cin, P, Cout,
                                              Cin, prec, _stream()), "usip_wgrad")
        torch.cuda.synchronize()
        out[prec] = gW.cpu().numpy().astype(np.float64)
    ref = G.wgrad_ref(GY, X)
    mag = G.err_bound(np.ascontiguousarray(GY.T), np.ascontiguousarray(X.T), 1.0)
    _check_bound("wgrad %s P=%d" % (path, P), out[1], out[4], ref, mag, G.TAU_WGRAD)


# ============================================================================ determinism
DET_CASES = [
    # id, P, Cin, Cout, prec, group, stats, path
    ("rowwarp", 1001, 256, 4, "fp32", 0, False, "rowwarp"),
    ("narrow1", 5000, 6, 32, "fp32", 0, True, "narrow1"),
    ("narrow2", 5000, 8, 64, "fp32", 0, True, "narrow2"),
    ("simt64", 5008, 100, 64, "fp32", 16, True, "simt64"),
    ("simt128", 5120, 100, 200, "fp32", 128, True, "simt128"),
    ("tc64", 4100, 96, 128, "3x", 0, True, "tc64"),
    ("tc64_g32", 4096, 96, 128, "3x", 32, True, "tc64"),
    ("tc128_g64", 17024, 256, 128, "3x", 64, True, "tc128"),
    ("tc128_combine", 16896, 256, 128, "3x", 128, True, "tc128+combine"),
    ("tc64_tf32", 4100, 96, 128, "tf32", 0, True, "tc64+tf32"),
]


@pytest.mark.parametrize("case", DET_CASES, ids=[c[0] for c in DET_CASES])
def test_layer_deterministic(case):
    """Two launches on the same Gaussian inputs: the same bits in Y, every statistic partial and the group outputs."""
    cid, P, Cin, Cout, prec, group, stats, path = case
    sm = sm_count()
    raw = path.startswith("narrow")
    assert G.layer_path(P, Cin, Cout, sm, precision=0 if prec == "fp32" else 1, single=prec == "tf32", stats=stats,
                        group=group, affine=not raw, relu=not raw) == path
    rng = np.random.default_rng(P + Cout)
    op = _upload(dict(bias=rng.normal(size=Cout).astype(np.float32),
                      scale=None if raw else rng.normal(size=Cin).astype(np.float32),
                      shift=None if raw else rng.normal(size=Cin).astype(np.float32), relu=not raw,
                      addend=None, add_index=None, add_group=None))
    X, W = Buf(rng.normal(size=(P, Cin)).astype(np.float32), Cin), Buf(rng.normal(size=(Cout, Cin)).astype(np.float32), Cin)
    runs = []
    for _ in range(2):
        Y = Buf(np.zeros((P, Cout), np.float32), Cout, fill=SENT)
        grp = None
        if group:
            Q = P // group
            grp = dict(g=group, gmax=torch.empty((Q, Cout), device="cuda"), gmin=torch.empty((Q, Cout), device="cuda"),
                       amax=torch.empty((Q, Cout), dtype=torch.int32, device="cuda"),
                       amin=torch.empty((Q, Cout), dtype=torch.int32, device="cuda"))
        ws = torch.empty(2 * Cin * Cout, device="cuda") if prec != "fp32" else None
        part = None
        if stats:
            part = torch.full((len(G.stat_slot_rows(path, P, Cout, sm)), 2, Cout), NAN, device="cuda")
        d = _layer_desc(P, Cin, Cout, X, W, False, op, Y, prec, part=part, grp=grp, ws=ws)
        _lib().check(_lib().load().usip_layer_fwd(ctypes.byref(d), _stream()), "usip_layer_fwd")
        torch.cuda.synchronize()
        outs = [Y.view().clone()] + ([part] if stats else []) + ([grp[k] for k in ("gmax", "gmin", "amax", "amin")] if group else [])
        runs.append([o.view(torch.int32) if o.dtype == torch.float32 else o for o in outs])
    for a, b in zip(*runs):
        assert torch.equal(a, b), cid
    if stats:
        assert not torch.isnan(runs[0][1].view(torch.float32)).any(), "unwritten statistic slot"
