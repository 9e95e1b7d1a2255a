"""Exact references for the layer GEMM (usip_layer_fwd) and the weight-gradient GEMM (usip_wgrad), in plain numpy.

Dyadic lattices.  When every operand, every product and every partial sum of a GEMM is a multiple of one step 2^-s and
stays below 2^24 steps, fp32 adds without rounding in any order: SIMT fma chains, warp shuffles, atomics and wgmma
accumulation all give the float64 sum bit for bit.  Two lattices are built here:
  * "int": small integers (and halves after a power-of-two BN prologue).  Every value is a TF32 value (lo == 0), so every
    precision gives the same exact answer; the test then pins data movement (rows, K chunks, strides, tails, prologue,
    bias, addend) and the group / statistic epilogues, ties included.
  * "lo_a" / "lo_w" (and "lo_gy" / "lo_x" for the weight gradient): one operand is m + n 2^-12 (a non-zero TF32 lo
    part), the other a TF32 value.  Then hi(a) hi(w) + hi(a) lo(w) + lo(a) hi(w) is the exact product, so fp32 and
    3xTF32 must equal the float64 reference, while plain TF32 must equal sum hi(a) hi(w), a different value: the output
    says which path ran and whether the compensation terms are there.

Also here: the per-element error bound of the non-lattice tests, and which kernel a layer / wgrad call reaches, restated
from the dispatch code (csrc/mlp.cu usip_layer_fwd, csrc/mlp_tc.cu tc_pick_bn, csrc/backward.cu usip_wgrad and
csrc/wgrad_tc.cu wgrad_tc) for a given SM count.
"""
import numpy as np

F32_EXACT = 2 ** 24          # integers of magnitude < 2^24 (in steps) are exact in fp32
LO = 2.0 ** -12              # the lo-lattice unit: below TF32's 10 mantissa bits at magnitude 1


# ----------------------------------------------------------------------------- TF32
def tf32(a):
    """cvt.rna.tf32.f32: round to nearest, ties away from zero, keeping 10 mantissa bits (finite inputs)."""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def split(a):
    """(hi, lo) = (rna_tf32(a), rna_tf32(a - hi)) with a - hi in fp32, as the kernels split an operand."""
    a = np.asarray(a, np.float32)
    hi = tf32(a)
    return hi, tf32(a - hi)


# ----------------------------------------------------------------------------- float64 restatements
def prologue(X, scale, shift, relu):
    """The folded BN prologue act(x) = relu(fmaf(x, scale, shift)) as fp32 values (x*scale is exact in float64)."""
    A = np.asarray(X, np.float64)
    if scale is not None:
        A = A * np.asarray(scale, np.float64) + np.asarray(shift, np.float64)
    A = A.astype(np.float32)
    return np.maximum(A, np.float32(0)) if relu else A


def _terms(A, W, mode):
    """[(a_part, w_part)] whose products the path sums: fp32 / 3xTF32 / plain TF32."""
    if mode == "fp32":
        return [(A, W)]
    (ah, al), (wh, wl) = split(A), split(W)
    if mode == "tf32":
        return [(ah, wh)]
    assert mode == "3x", mode
    return [(al, wh), (ah, wl), (ah, wh)]


def layer_ref(A, W, bias=None, add_rows=None, mode="fp32"):
    """Y[P, Cout] = sum_k A[p,k] W[n,k] (+ bias + addend row) in float64; A are the activations after the prologue,
    W is [Cout, Cin].  mode picks the products the kernel forms (see _terms)."""
    Y = sum(np.asarray(a, np.float64) @ np.asarray(w, np.float64).T for a, w in _terms(A, W, mode))
    if bias is not None:
        Y = Y + np.asarray(bias, np.float64)
    if add_rows is not None:
        Y = Y + np.asarray(add_rows, np.float64)
    return Y


def wgrad_ref(GY, A, gW0=None, mode="fp32"):
    """gW0 + GY^T A in float64 ([Cout, Cin]); GY is the A operand of the kernel's GEMM, act(X) the B operand."""
    G = sum(np.asarray(g, np.float64).T @ np.asarray(a, np.float64) for g, a in _terms(GY, A, mode))
    return G if gW0 is None else G + np.asarray(gW0, np.float64)


def group_ref(Y, g):
    """Per-group max / min over g consecutive rows and the row-in-group of each: ties go to the FIRST row."""
    Yg = np.asarray(Y).reshape(-1, g, Y.shape[1])
    return Yg.max(1), Yg.min(1), Yg.argmax(1).astype(np.int32), Yg.argmin(1).astype(np.int32)


def abs_sum(A, W, mode="fp32"):
    """sum_k |a_k| |w_k| over the products the path forms: bounds every partial sum of the dot product, in any order."""
    return sum(np.abs(np.asarray(a, np.float64)) @ np.abs(np.asarray(w, np.float64)).T for a, w in _terms(A, W, mode))


def on_lattice(vals, step):
    v = np.asarray(vals, np.float64) / step
    return bool(np.all(v == np.round(v)))


def exact_premise(terms, extra, step):
    """Checks that every addend in `extra` is a multiple of `step` and returns the bound, in steps, on every partial sum
    of the GEMM over `terms` ([(a [M,K], b [N,K])]): sum over the terms of |a||b| plus |extra|.  With every product a
    multiple of step (products_on_lattice), fp32 is exact on the GEMM when the bound is below 2^24."""
    bound = 0.0
    for a, b in terms:
        bound = bound + np.abs(np.asarray(a, np.float64)) @ np.abs(np.asarray(b, np.float64)).T
    for e in extra:
        if e is not None:
            assert on_lattice(e, step), "addend off the lattice"
            bound = bound + np.abs(np.asarray(e, np.float64))
    return float(np.max(bound)) / step


def products_on_lattice(A, W, step, mode):
    """Every product a_k w_k the path forms is a multiple of step (checked on the distinct operand values)."""
    for a, w in _terms(A, W, mode):
        av = np.unique(np.asarray(a, np.float64)); wv = np.unique(np.asarray(w, np.float64))
        if not on_lattice(np.outer(av, wv), step):
            return False
    return True


def err_bound(A, W, tau, extra=(), mode="fp32"):
    """Per-element error bound tau * (sum_k |a_k| |w_k| + |bias| + |addend|) of the non-lattice tests."""
    b = abs_sum(A, W, mode)
    for e in extra:
        if e is not None:
            b = b + np.abs(np.asarray(e, np.float64))
    return tau * b


# ----------------------------------------------------------------------------- lattice operands
def _pick(rng, vals, shape):
    return np.asarray(vals, np.float32)[rng.integers(0, len(vals), size=shape)]


def _lo_vals(rng, shape, zeros=1):
    """m + n 2^-12, m in {-1, 0 (x zeros), 1}, n in {-1, 1}: the hi part is m (or n 2^-12 when m == 0), the lo part
    +-2^-12 when m != 0 (for m = -1, n = +1 the magnitude 1 - 2^-12 sits on a TF32 tie and rounds away to 1)."""
    m = _pick(rng, [-1.0] + [0.0] * zeros + [1.0], shape)
    n = _pick(rng, [-1.0, 1.0], shape)
    return (m + n * np.float32(LO)).astype(np.float32)


def tie_rows(rng, P, g):
    """Row map for duplicated rows inside groups of g: in every other group, rows are copies of a few prototype rows whose
    first copies sit at offsets 0, 3, 17, 35, 66 and 100 (inside a 4-row chunk, past the 16-row segment, the 32-row quarter,
    the 64-row warpgroup tile), and every later row repeats one prototype already seen.  The ties of max and min are then
    decided across every boundary of the SIMT and wgmma epilogues.  Returns src[P]: row r takes the data of row src[r]."""
    src = np.arange(P)
    firsts = [f for f in (0, 3, 17, 35, 66, 100) if f < g]
    for q in range(0, P // g, 2):
        base = q * g
        seen = []
        for r in range(g):
            if r in firsts:
                seen.append(base + r)
            else:
                src[base + r] = seen[rng.integers(0, len(seen))]
    return src


def layer_operands(seed, P, Cin, Cout, kind="int", prologue_kind="affine_relu", addend=None, n_add=37, wdens=1.0,
                   ties=0):
    """Lattice operands of one usip_layer_fwd call.  kind: "int", "lo_a" (activation side carries the lo part: through the
    BN scale with a prologue, in X itself without), "lo_w" (weight side).  prologue_kind: "affine_relu", "affine", "relu"
    or "none".  addend: None, "index" or "group".  ties > 0 duplicates rows inside groups of `ties` rows (tie_rows)."""
    rng = np.random.default_rng(seed)
    affine = prologue_kind.startswith("affine")
    relu = prologue_kind in ("affine_relu", "relu")
    scale = shift = None
    if kind == "int":
        X = _pick(rng, [-2, -1, 0, 1, 2], (P, Cin))
        W = _pick(rng, [-3, -2, -1, 1, 2, 3], (Cout, Cin)) * (rng.random((Cout, Cin)) < wdens)
        if affine:
            scale = _pick(rng, [-2, -1, -0.5, 0.5, 1, 2], Cin)
            shift = _pick(rng, [-1, -0.5, 0, 0.5, 1], Cin)
        step = 0.5 if affine else 1.0
    elif kind == "lo_w":
        X = _pick(rng, [-1, 0, 1], (P, Cin))
        W = _lo_vals(rng, (Cout, Cin), zeros=2) * (rng.random((Cout, Cin)) < wdens)
        if affine:
            scale = _pick(rng, [-1, 1], Cin); shift = _pick(rng, [0, 1], Cin)
        step = LO
    elif kind == "lo_a":
        W = _pick(rng, [-1, 0, 1], (Cout, Cin)) * (rng.random((Cout, Cin)) < wdens)
        if affine:
            X = _pick(rng, [-1, 0, 1], (P, Cin))
            scale = (_pick(rng, [-1, 1], Cin) * (1 + _pick(rng, [-1, 1], Cin) * np.float32(LO))).astype(np.float32)
            shift = np.zeros(Cin, np.float32)
        else:
            X = _lo_vals(rng, (P, Cin))
        step = LO
    else:
        raise ValueError(kind)
    W = W.astype(np.float32)
    bias = _pick(rng, [-4, -2, -1, 0, 1, 3], Cout)
    add_index = add_group = add = None
    if addend == "index":
        G = n_add
        add_index = rng.integers(0, G, size=P).astype(np.int32)
        if ties:
            add_index = rng.integers(0, G, size=-(-P // ties)).astype(np.int32)[np.arange(P) // ties]
    elif addend == "group":
        add_group = ties if ties else 64
        G = -(-P // add_group)
    if addend:
        add = _pick(rng, [-3, -1, 0, 1, 2], (G, Cout))
    if ties:
        X = X[tie_rows(rng, P, ties)]
    A = prologue(X, scale, shift, relu)
    add_rows = None
    if addend == "index":
        add_rows = add[add_index]
    elif addend == "group":
        add_rows = add[np.arange(P) // add_group]
    return dict(X=X, W=W, bias=bias, scale=scale, shift=shift, relu=relu, addend=add, add_index=add_index,
                add_group=add_group, add_rows=add_rows, A=A, step=step, kind=kind)


def layer_premise(op, modes=("fp32", "3x", "tf32")):
    """The exactness premise of a layer lattice case: every product a multiple of the step, every partial sum below 2^24
    steps, for every mode the case is compared in.  Returns the largest bound in steps."""
    worst = 0.0
    for mode in modes:
        assert products_on_lattice(op["A"], op["W"], op["step"], mode), mode
        worst = max(worst, exact_premise(_terms(op["A"], op["W"], mode), (op["bias"], op["add_rows"]), op["step"]))
    return worst


def layer_expect(op, mode):
    return layer_ref(op["A"], op["W"], op["bias"], op["add_rows"], mode)


def stat_slot_rows(path, P, Cout, sm):
    """The rows whose (sum y, sum y^2) each BN-statistic partial row holds, restated from the kernels: one slot per
    128-row tile for the fp32 kernels; for the persistent tensor-core kernel one slot per (CTA row base, warpgroup,
    32-row quarter), slot base*4 + 2 wg + q, accumulated over the warpgroup's tiles base + k stride (mlp_tc.cu)."""
    if not path.startswith("tc"):
        return [np.arange(t, min(t + 128, P)) for t in range(0, P, 128)]
    bn = 128 if path.startswith("tc128") else 64
    combine = "+combine" in path
    n_tiles = Cout // bn
    grid = max(n_tiles, min(sm, _cdiv(P, 128) * n_tiles) // n_tiles * n_tiles)
    stride = grid // n_tiles
    tile_rows = 128 if combine else 64
    slots = []
    for base in range(stride):
        cta_tiles = _cdiv(_cdiv(P, tile_rows) - base, stride)
        for wg in range(2):
            n_wg = cta_tiles if combine else (cta_tiles + 1 - wg) // 2
            starts = [((base + jt * stride) * 128 + 64 * wg) if combine else (base + (2 * jt + wg) * stride) * 64
                      for jt in range(n_wg)]
            for q in range(2):
                rows = [np.arange(s + 32 * q, min(s + 32 * q + 32, P)) for s in starts]
                slots.append(np.concatenate(rows) if rows else np.zeros(0, np.int64))
    return slots


def stats_ref(Y, slots):
    """[slots, 2, Cout] float64 (sum y, sum y^2) over each slot's rows."""
    Y = np.asarray(Y, np.float64)
    out = np.zeros((len(slots), 2, Y.shape[1]))
    for i, r in enumerate(slots):
        out[i, 0] = Y[r].sum(0); out[i, 1] = (Y[r] ** 2).sum(0)
    return out


def stats_exact(Y, step, slots=None):
    """Whether every fp32 partial (sum y, sum y^2) a slot accumulates is exact: the slot totals of |y| and y^2 stay
    below 2^24 steps (step and step^2).  slots=None: the whole of Y as one slot."""
    Y = np.abs(np.asarray(Y, np.float64))
    slots = [np.arange(Y.shape[0])] if slots is None else slots
    S = stats_ref(Y, slots)
    return bool(S[:, 0].max() / step < F32_EXACT and S[:, 1].max() / step ** 2 < F32_EXACT)


def wgrad_operands(seed, P, Cout, Cin, kind="int", prologue_kind="affine_relu"):
    """Lattice operands of one usip_wgrad call: GY [P, Cout], X [P, Cin] (+ BN prologue), gW0 [Cout, Cin] (the += base).
    kind: "int", "lo_gy" (the GEMM's A operand carries the lo part) or "lo_x" (act(X), through the BN scale with an
    affine prologue, in X itself without).  The lo kinds are half zeros so that sums over thousands of rows stay exact."""
    rng = np.random.default_rng(seed)
    affine = prologue_kind.startswith("affine")
    relu = prologue_kind in ("affine_relu", "relu")
    scale = shift = None
    if kind == "int":
        GY = _pick(rng, [-2, -1, 0, 1, 2], (P, Cout))
        X = _pick(rng, [-2, -1, 0, 1, 2], (P, Cin))
        if affine:
            scale = _pick(rng, [-2, -1, -0.5, 0.5, 1, 2], Cin); shift = _pick(rng, [-1, -0.5, 0, 0.5, 1], Cin)
        step = 0.5 if affine else 1.0
    elif kind == "lo_gy":
        GY = _lo_vals(rng, (P, Cout), zeros=4)
        X = _pick(rng, [-1, 0, 0, 1], (P, Cin))
        if affine:
            scale = _pick(rng, [-1, 1], Cin); shift = np.zeros(Cin, np.float32)
        step = LO
    elif kind == "lo_x":
        GY = _pick(rng, [-1, 0, 0, 1], (P, Cout))
        if affine:
            X = _pick(rng, [-1, 0, 0, 1], (P, Cin))
            scale = (_pick(rng, [-1, 1], Cin) * (1 + _pick(rng, [-1, 1], Cin) * np.float32(LO))).astype(np.float32)
            shift = np.zeros(Cin, np.float32)
        else:
            X = _lo_vals(rng, (P, Cin), zeros=4)
        step = LO
    else:
        raise ValueError(kind)
    gW0 = _pick(rng, [-8, -1, 0, 1, 5], (Cout, Cin))
    A = prologue(X, scale, shift, relu)
    return dict(GY=GY, X=X, scale=scale, shift=shift, relu=relu, A=A, gW0=gW0, step=step, kind=kind)


def wgrad_premise(op, modes=("fp32", "3x", "tf32")):
    worst = 0.0
    for mode in modes:
        GYt = np.ascontiguousarray(op["GY"].T); At = np.ascontiguousarray(op["A"].T)
        assert products_on_lattice(GYt, At, op["step"], mode), mode
        worst = max(worst, exact_premise(_terms(GYt, At, mode), (op["gW0"],), op["step"]))
    return worst


def wgrad_expect(op, mode):
    return wgrad_ref(op["GY"], op["A"], op["gW0"], mode)


# ----------------------------------------------------------------------------- dispatch restatement
def _cdiv(a, b):
    return -(-a // b)


ROWWARP_SMEM = 48 * 1024


def layer_path(P, Cin, Cout, sm, precision=0, single=False, stats=False, group=0, addend=False, affine=False,
               relu=False):
    """The kernel usip_layer_fwd launches for a descriptor (group > 0: gmax / gmin requested).
    precision 1: "tc64" / "tc128" (column-tile width, tc_pick_bn), "+combine" for the group-128 combine, "+tf32" for the
    plain TF32 option.  precision 0: "rowwarp", "narrow1" / "narrow2" (32 / 64 channels per CTA pass), "simt64" / "simt128"."""
    if precision == 1:
        bn = 128 if Cout % 128 == 0 and _cdiv(P, 128) * (Cout // 128) >= sm else 64
        return "tc%d" % bn + ("+combine" if group == 128 else "") + ("+tf32" if single else "")
    if Cout <= 8 and not stats and not group and not addend and (8 + 2) * Cin * 4 <= ROWWARP_SMEM:
        return "rowwarp"
    if Cin <= 8 and Cout in (32, 64) and not affine and not relu and not addend and not group:
        return "narrow2" if Cout == 64 else "narrow1"
    return "simt64" if Cout <= 64 else "simt128"


def wgrad_path(P, Cout, Cin, precision, ldg=None, ldx=None, gy_aligned=True, x_aligned=True, affine_aligned=True):
    """The kernel usip_wgrad launches: "tc64" / "tc128" (+"+tf32" at precision 4), "narrow" or "simt".  An ineligible
    precision 1 or 4 call runs the fp32 kernels."""
    ldg = Cout if ldg is None else ldg
    ldx = Cin if ldx is None else ldx
    if precision in (1, 4):
        ok = (Cout % 4 == 0 and Cout >= 64 and Cin % 64 == 0 and P >= 4096 and ldg % 4 == 0 and ldx % 4 == 0
              and gy_aligned and x_aligned and affine_aligned)
        if ok:
            return ("tc128" if Cin % 128 == 0 else "tc64") + ("+tf32" if precision == 4 else "")
    if Cin <= 8 and Cout in (32, 64, 128, 256) and P >= 4096 and ldg % 4 == 0 and gy_aligned:
        return "narrow"
    return "simt"


def wgrad_simt_split(P, Cout, Cin, sm):
    """(CTAs along P, rows per CTA) of the fp32 SIMT wgrad kernel."""
    tiles = _cdiv(Cout, 128) * _cdiv(Cin, 128)
    splits = max(1, min(_cdiv(P, 128), (sm * 4) // tiles))
    rows = _cdiv(_cdiv(P, splits), 16) * 16
    return _cdiv(P, rows), rows


# ----------------------------------------------------------------------------- the lattice cases of the GPU tests
def case_seed(cid):
    return sum((i + 1) * ord(c) for i, c in enumerate(cid)) % 2 ** 31


# Layer cases: (id, P, Cin, Cout, kwargs).  kwargs: kind, pro (prologue), add (addend mode), stats, group, args, prec
# ("fp32" | "3x" | "tf32"), ldx_pad, x_off / w_off (a float off 16-byte alignment), wt (W stored [Cin, Cout]), ldw_pad,
# ldy_pad, ties, wdens, path (the kernel the case is written for, on a 132-SM H100 SXM).
def _c(cid, P, Cin, Cout, path, **kw):
    kw.setdefault("kind", "int"); kw.setdefault("pro", "affine_relu"); kw.setdefault("prec", "fp32")
    kw["path"] = path
    return (cid, P, Cin, Cout, kw)


LAYER_CASES = [
    # ---- row-warp head kernel (Cout <= 8): Cin at the 48 KB shared-memory limit and one past it, P % 8 != 0
    _c("rowwarp_cout1", 1001, 200, 1, "rowwarp", ldx_pad=3, ldy_pad=2),
    _c("rowwarp_cout4_lo_a", 1003, 256, 4, "rowwarp", kind="lo_a", wt=True, ldw_pad=3),
    _c("rowwarp_cout8_lo_w", 517, 96, 8, "rowwarp", kind="lo_w", pro="relu", ldx_pad=1, ldy_pad=1),
    _c("rowwarp_cin1228", 333, 1228, 8, "rowwarp", ldx_pad=4),
    _c("rowwarp_cin1229_simt", 333, 1229, 8, "simt64", ldx_pad=4),
    # ---- narrow first-layer kernel: Cin 1..8, scalar (ldx < 8) and vector (ldx >= 8, aligned) loads, transposed W
    _c("narrow1_cin1_ldx1", 1000, 1, 32, "narrow1", pro="none", stats=True),
    _c("narrow2_cin2_ldx8", 1100, 2, 64, "narrow2", pro="none", ldx_pad=6, stats=True),
    _c("narrow1_cin3_ldx8_wt", 1000, 3, 32, "narrow1", pro="none", ldx_pad=5, wt=True, ldw_pad=3),
    _c("narrow2_cin4_lo_a", 4133, 4, 64, "narrow2", kind="lo_a", pro="none", ldx_pad=4),
    _c("narrow1_cin5_ldx5", 777, 5, 32, "narrow1", pro="none", stats=True),
    _c("narrow2_cin6_ldx12_lo_w", 1000, 6, 64, "narrow2", kind="lo_w", pro="none", ldx_pad=6, wt=True),
    _c("narrow1_cin7_ldx8", 4200, 7, 32, "narrow1", pro="none", ldx_pad=1, stats=True),
    _c("narrow2_cin8_ldx8", 1000, 8, 64, "narrow2", pro="none", stats=True),
    _c("narrow2_cin7_unaligned", 640, 7, 64, "narrow2", pro="none", ldx_pad=1, x_off=1, stats=True),
    # ---- SIMT<64> / SIMT<128>: Cin % 8 != 0, ldx % 4 != 0, views off alignment, Cout % 4 != 0, groups 4..128, P tails
    _c("simt64_cin37_cout30", 1000, 37, 30, "simt64", ldx_pad=2, stats=True, add="index"),
    _c("simt64_unaligned_lo_a", 1000, 36, 60, "simt64", kind="lo_a", x_off=1, w_off=1, ldx_pad=1, ldw_pad=3),
    _c("simt128_cin36_cout130_wt", 999, 36, 130, "simt128", wt=True, ldw_pad=2, stats=True, add="group"),
    _c("simt128_lo_w_unaligned", 700, 100, 100, "simt128", kind="lo_w", w_off=1, x_off=1, ldy_pad=3),
    _c("simt64_g4", 1000, 24, 64, "simt64", group=4, args=True, ties=4, stats=True, add="index"),
    _c("simt64_g8_relu", 1000, 20, 48, "simt64", pro="relu", group=8, args=True, ties=8, stats=True),
    _c("simt128_g16", 960, 44, 128, "simt128", group=16, args=True, ties=16, stats=True, add="group"),
    _c("simt128_g32", 960, 72, 100, "simt128", group=32, args=True, ties=32, stats=True, x_off=1, ldx_pad=1),
    _c("simt64_g64", 960, 40, 64, "simt64", group=64, args=True, ties=64, stats=True, add="index"),
    _c("simt128_g128", 1024, 52, 256, "simt128", group=128, args=True, ties=128, stats=True, add="group"),
    _c("simt128_g128_lo_w", 1024, 52, 130, "simt128", kind="lo_w", group=128, args=True, ties=128),
    # ---- tensor cores: width 64 / 128, COMBINE or not, 3xTF32 and plain TF32
    _c("tc64_one_chunk", 5000, 32, 64, "tc64", prec="3x", stats=True, add="index"),
    _c("tc64_tail17", 4113, 64, 64, "tc64", prec="3x", stats=True, add="index", ldx_pad=4),
    _c("tc64_ring_lo_a", 3000, 320, 64, "tc64", prec="3x", kind="lo_a"),
    _c("tc64_ring_lo_a_tf32", 3000, 320, 64, "tc64+tf32", prec="tf32", kind="lo_a"),
    _c("tc128_ring_tail", 16996, 256, 256, "tc128", prec="3x", stats=True, wdens=0.0625, add="index"),
    _c("tc128_ring_lo_w", 16996, 256, 256, "tc128", prec="3x", kind="lo_w", ldx_pad=8),
    _c("tc128_ring_lo_w_tf32", 16996, 256, 256, "tc128+tf32", prec="tf32", kind="lo_w", ldx_pad=8),
    _c("tc128_uneven_wgs", 17000, 256, 128, "tc128", prec="3x", stats=True, wdens=0.0625, add="group"),
    _c("tc64_empty_wg", 192, 64, 64, "tc64", prec="3x", stats=True),
    _c("tc64_one_tile", 40, 96, 128, "tc64", prec="3x", stats=True, add="index"),
    _c("tc64_one_tile_lo_a_tf32", 40, 96, 128, "tc64+tf32", prec="tf32", kind="lo_a"),
    _c("tc64_wt_lo_w", 4100, 64, 128, "tc64", prec="3x", kind="lo_w", wt=True, ldw_pad=4),
    _c("tc128_wt_lo_w_tf32", 17000, 256, 256, "tc128+tf32", prec="tf32", kind="lo_w", wt=True),
    _c("tc128_g16", 16512, 64, 256, "tc128", prec="3x", group=16, ties=16, stats=True, add="index"),
    _c("tc64_g32", 4160, 160, 128, "tc64", prec="3x", group=32, ties=32, stats=True, add="group"),
    _c("tc128_g64", 17024, 512, 128, "tc128", prec="3x", group=64, ties=64, stats=True, wdens=0.03),
    _c("tc128_g128", 16896, 256, 128, "tc128+combine", prec="3x", group=128, ties=128, stats=True, wdens=0.0625,
       add="index"),
    _c("tc64_g128", 8192, 96, 64, "tc64+combine", prec="3x", group=128, ties=128, stats=True, add="group"),
    _c("tc64_g128_tf32_lo_a", 8192, 96, 64, "tc64+combine+tf32", prec="tf32", kind="lo_a", group=128, ties=128),
    _c("tc64_g64_tf32_lo_w", 4096, 128, 128, "tc64+tf32", prec="tf32", kind="lo_w", group=64, ties=64, ldx_pad=4),
]

# wgrad cases: (id, P, Cout, Cin, kwargs): kind, pro, prec (usip_wgrad precision 0 / 1 / 4), ldx_pad, ldg_pad,
# gy_off / x_off, ldw_pad, path
def _w(cid, P, Cout, Cin, path, **kw):
    kw.setdefault("kind", "int"); kw.setdefault("pro", "affine_relu"); kw.setdefault("prec", 1)
    kw["path"] = path
    return (cid, P, Cout, Cin, kw)


WGRAD_CASES = [
    # ---- narrow kernel (Cin <= 8, Cout in {32, 64, 128, 256}, P >= 4096): packed ldx == 8 and a generic ldx
    _w("narrow_cout32_cin3_ldx8", 4096, 32, 3, "narrow", prec=0, ldx_pad=5),
    _w("narrow_cout64_cin8_lo_gy", 5000, 64, 8, "narrow", kind="lo_gy", prec=4),
    _w("narrow_cout128_cin5_lo_x", 4500, 128, 5, "narrow", kind="lo_x", pro="none", prec=1, ldx_pad=2, ldw_pad=3),
    _w("narrow_cout256_cin7_ldx8", 4096, 256, 7, "narrow", prec=1, ldx_pad=1),
    _w("narrow_p4095_simt", 4095, 64, 8, "simt", prec=1),
    # ---- fp32 SIMT kernel, split over P: the last CTA's slice a single row, or exactly full
    _w("simt_split_tail1", None, 100, 100, "simt", prec=0, split="tail1", ldg_pad=1, ldx_pad=3),
    _w("simt_split_full", None, 100, 100, "simt", prec=0, split="full", kind="lo_x"),
    _w("simt_cout6_cin131", 3000, 6, 131, "simt", prec=1, kind="lo_gy", ldw_pad=5),
    # ---- tensor cores: width 128 (Cin % 128 == 0) and 64, Cout 64 and 100 (a partial 128-channel tile), P edges
    _w("tc128_cout64", 4096, 64, 128, "tc128", kind="lo_gy", ldw_pad=4),
    _w("tc128_cout64_tf32", 4096, 64, 128, "tc128+tf32", prec=4, kind="lo_gy"),
    _w("tc128_p4095_simt_tf32", 4095, 64, 128, "simt", prec=4, kind="lo_gy"),
    _w("tc64_cout100", 4113, 100, 192, "tc64", kind="lo_x", ldx_pad=4, ldw_pad=2),
    _w("tc64_cout100_tf32", 4113, 100, 192, "tc64+tf32", prec=4, kind="lo_x", ldx_pad=4),
    _w("tc64_cout100_int", 4096 + 17, 100, 64, "tc64", ldg_pad=4, ldw_pad=1),
    _w("tc128_tail_tf32_lo_x", 5000 + 9, 128, 256, "tc128+tf32", prec=4, kind="lo_x", pro="relu"),
    _w("tc_unaligned_gy_tf32", 4096, 64, 128, "simt", prec=4, kind="lo_gy", gy_off=1),
    _w("tc_unaligned_x_tf32", 4096, 64, 128, "simt", prec=4, kind="lo_x", x_off=1),
    _w("tc_ldx_odd_tf32", 4096, 64, 128, "simt", prec=4, kind="lo_x", ldx_pad=1),
]


def wgrad_case_P(P, Cout, Cin, kw, sm):
    """P of a case: given, or chosen against the SIMT split so that the last CTA's slice is one row ("tail1") or exactly
    full ("full")."""
    if P is not None:
        return P
    for p in range(3000, 9000):
        splits, rows = wgrad_simt_split(p, Cout, Cin, sm)
        r = p - (splits - 1) * rows
        if splits > 1 and r == (1 if kw["split"] == "tail1" else rows):
            return p
    raise AssertionError("no P for split %s" % kw["split"])


# ----------------------------------------------------------------------------- the error-bound cases (off the lattice)
# tau of the per-element bound |y - y64| <= tau * (sum_k |a_k| |w_k| + |bias|) of the 3xTF32 kernels.  The wgmma
# accumulators do not round to nearest: the layer's worst error measured on an H100 80GB HBM3 (SXM, 700 W), 1.18e-6 at
# K = 256 (three wgmma per k-step of 8, 96 accumulations), lies between this module's model of round-to-nearest
# accumulation (4.5e-7) and of round-toward-zero accumulation (1.6e-6, layer_3x_truncating), so 4x the measured value
# does not fit under 2^-18 and the layer bound is 2^-17.  The weight gradient measured 3.1e-7.
TAU_LAYER = 2.0 ** -17
TAU_WGRAD = 2.0 ** -19


def _z(rng, shape):
    """N(0, 1) with |z| >= 1/64: scaled by 2^+-48 at most, no operand or product comes near the subnormals."""
    z = rng.normal(size=shape)
    return np.sign(z) * np.maximum(np.abs(z), 1 / 64)


def bound_layer_operands(P, Cin, Cout):
    """X [P, Cin], W [Cout, Cin], bias: row scales 2^[-20, 20], output-column scales 2^[-20, 20], K-chunk scales
    2^[-8, 8] on each operand."""
    rng = np.random.default_rng(P + Cin)
    e_p, f_n = rng.integers(-20, 21, P), rng.integers(-20, 21, Cout)
    g_k, h_k = rng.integers(-8, 9, Cin // 32).repeat(32), rng.integers(-8, 9, Cin // 32).repeat(32)
    X = (_z(rng, (P, Cin)) * np.exp2(e_p[:, None] + g_k[None, :])).astype(np.float32)
    W = (_z(rng, (Cout, Cin)) * np.exp2(f_n[:, None] + h_k[None, :])).astype(np.float32)
    return X, W, (_z(rng, Cout) * np.exp2(f_n)).astype(np.float32)


def bound_wgrad_operands(P, Cout, Cin):
    """GY [P, Cout], X [P, Cin]: 32-row chunk scales 2^[-10, 10] on each operand, output-row and -column scales
    2^[-20, 20]."""
    rng = np.random.default_rng(P + Cout)
    e_r = rng.integers(-10, 11, -(-P // 32)).repeat(32)[:P]
    e2_r = rng.integers(-10, 11, -(-P // 32)).repeat(32)[:P]
    f_m, g_j = rng.integers(-20, 21, Cout), rng.integers(-20, 21, Cin)
    GY = (_z(rng, (P, Cout)) * np.exp2(e_r[:, None] + f_m[None, :])).astype(np.float32)
    X = (_z(rng, (P, Cin)) * np.exp2(e2_r[:, None] + g_j[None, :])).astype(np.float32)
    return GY, X


def _round_toward_zero(x64):
    x32 = x64.astype(np.float32)
    over = np.abs(x32.astype(np.float64)) > np.abs(x64)
    return np.where(over, np.nextafter(x32, np.float32(0)), x32)


def layer_3x_truncating(A, W, bias=None):
    """Model of the 3xTF32 layer kernel's arithmetic: per k-step of 8, the exact sums of lo*hi, hi*lo and hi*hi each added
    to an fp32 accumulator that rounds toward zero, then + bias."""
    (ah, al), (wh, wl) = split(A), split(W)
    acc = np.zeros((A.shape[0], W.shape[0]), np.float32)
    for k in range(0, A.shape[1], 8):
        s = slice(k, k + 8)
        for a, w in ((al, wh), (ah, wl), (ah, wh)):
            acc = _round_toward_zero(acc.astype(np.float64) + a[:, s].astype(np.float64) @ w[:, s].astype(np.float64).T)
    y = acc if bias is None else acc + np.asarray(bias, np.float32)
    return y.astype(np.float64)
