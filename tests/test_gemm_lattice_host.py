"""CPU checks of the premises of tests/test_gpu_gemm_lattice.py: every lattice case is exact in fp32 in any summation
order, the TF32 split is cvt.rna.tf32.f32, plain TF32 is told apart from fp32 on every lo-lattice case, and the dispatch
restatement picks the documented kernel on both sides of every limit."""
import numpy as np
import pytest

from tests import gemm_ref as G

H100_SXM, H100_PCIE = 132, 114


# ----------------------------------------------------------------------------- lattice premises
@pytest.mark.parametrize("case", G.LAYER_CASES, ids=[c[0] for c in G.LAYER_CASES])
def test_layer_lattice_premise(case):
    cid, P, Cin, Cout, kw = case
    op = G.layer_operands(G.case_seed(cid), P, Cin, Cout, kw["kind"], kw["pro"],
                          kw.get("add"), wdens=kw.get("wdens", 1.0), ties=kw.get("ties", 0))
    bound = G.layer_premise(op)
    assert bound < G.F32_EXACT, (cid, bound)
    ref = G.layer_expect(op, "fp32")
    assert np.array_equal(ref.astype(np.float32).astype(np.float64), ref)
    # the compensated product is exact on a lattice whose lo parts sit on one side only
    assert np.array_equal(G.layer_expect(op, "3x"), ref)
    if kw["kind"] != "int":
        tf = G.layer_expect(op, "tf32")
        frac = float((tf != ref).mean())
        assert frac > 0.25, (cid, frac)
    else:
        lo = [G.split(a)[1] for a in (op["A"], op["W"])]
        assert not lo[0].any() and not lo[1].any()
    if kw.get("stats"):
        slots = G.stat_slot_rows(kw["path"], P, Cout, H100_SXM)
        assert np.array_equal(np.sort(np.concatenate(slots)), np.arange(P))     # every row in exactly one slot
        assert G.stats_exact(ref, op["step"], slots), cid
    if kw.get("group"):
        Yg = ref.reshape(-1, kw["group"], Cout)
        mx = Yg.max(1, keepdims=True)
        ties = ((Yg == mx).sum(1) > 1).mean()
        assert ties > 0.2, (cid, ties)      # the group max is decided between equal rows in many columns


@pytest.mark.parametrize("case", G.WGRAD_CASES, ids=[c[0] for c in G.WGRAD_CASES])
def test_wgrad_lattice_premise(case):
    cid, P, Cout, Cin, kw = case
    P = G.wgrad_case_P(P, Cout, Cin, kw, H100_SXM)
    op = G.wgrad_operands(G.case_seed(cid), P, Cout, Cin, kw["kind"], kw["pro"])
    bound = G.wgrad_premise(op)
    assert bound < G.F32_EXACT, (cid, bound)
    ref = G.wgrad_expect(op, "fp32")
    assert np.array_equal(ref.astype(np.float32).astype(np.float64), ref)
    assert np.array_equal(G.wgrad_expect(op, "3x"), ref)
    if kw["kind"] != "int":
        frac = float((G.wgrad_expect(op, "tf32") != ref).mean())
        assert frac > 0.25, (cid, frac)


# ----------------------------------------------------------------------------- TF32 split
def _rna_ref(x):
    """Independent restatement of round-to-nearest, ties away, to 11 significant bits, in float64."""
    x = np.asarray(x, np.float64)
    m, e = np.frexp(np.abs(x))                                     # |x| = m 2^e, m in [0.5, 1)
    q = np.floor(m * 2 ** 11 + 0.5)                                # 11 significant bits, ties away from zero
    return (np.sign(x) * np.ldexp(q, e - 11)).astype(np.float32)


def test_tf32_rna_matches_restatement():
    rng = np.random.default_rng(3)
    x = (rng.normal(size=20000) * np.exp2(rng.integers(-40, 40, size=20000))).astype(np.float32)
    # exact ties (the 13 dropped bits are 1000...0) and values just below / above them
    b = x.view(np.uint32) & np.uint32(0xffffe000)
    ties = (b | np.uint32(0x1000)).view(np.float32)
    near = np.concatenate([(b | np.uint32(0x0fff)).view(np.float32), (b | np.uint32(0x1001)).view(np.float32)])
    for v in (x, ties, near, np.float32([1 - 2 ** -12, -(1 - 2 ** -12), 1 + 2 ** -12, 2 ** -12])):
        assert np.array_equal(G.tf32(v), _rna_ref(v))
    assert G.tf32(np.float32([1 - 2 ** -12]))[0] == 1.0            # the tie rounds away from zero


def test_split_round_trips_on_the_lattices():
    rng = np.random.default_rng(5)
    vals = np.concatenate([G._lo_vals(rng, 4096), np.arange(-64, 65, dtype=np.float32) * 0.5,
                           (np.float32(1) + G._pick(rng, [-1, 1], 64) * np.float32(G.LO)) * G._pick(rng, [-1, 1], 64)])
    hi, lo = G.split(vals)
    assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), vals.astype(np.float64))
    assert np.array_equal(G.tf32(hi), hi) and np.array_equal(G.tf32(lo), lo)
    assert (lo[:4096] != 0).mean() > 0.4                          # the lo lattice really has lo parts
    # off the lattice the split drops at most the bits below 2^-21 of |x| (what 3xTF32 loses besides lo*lo)
    x = (rng.normal(size=4096) * np.exp2(rng.integers(-20, 20, size=4096))).astype(np.float32)
    hi, lo = G.split(x)
    d = np.abs(x.astype(np.float64) - hi - lo)
    assert np.all(d <= np.abs(x) * 2.0 ** -21)


# ----------------------------------------------------------------------------- dispatch restatement
@pytest.mark.parametrize("sm", [H100_SXM, H100_PCIE])
def test_layer_dispatch_edges(sm):
    L = G.layer_path
    # row-warp head: Cout <= 8, (8 + 2) Cin floats of shared memory <= 48 KB, no statistics / groups / addend
    assert L(1001, 1228, 8, sm) == "rowwarp" and L(1001, 1229, 8, sm) == "simt64"
    assert L(1001, 64, 1, sm) == "rowwarp" and L(1001, 64, 9, sm) == "simt64"
    assert L(1001, 64, 4, sm, stats=True) == "simt64" and L(1001, 64, 4, sm, group=4) == "simt64"
    assert L(1001, 64, 4, sm, addend=True) == "simt64"
    # narrow first layer: Cin <= 8, Cout 32 / 64, raw input, no addend / groups
    assert L(1000, 8, 32, sm) == "narrow1" and L(1000, 8, 64, sm, stats=True) == "narrow2"
    assert L(1000, 9, 64, sm) == "simt64" and L(1000, 8, 48, sm) == "simt64" and L(1000, 8, 128, sm) == "simt128"
    assert L(1000, 3, 32, sm, affine=True) == "simt64" and L(1000, 3, 32, sm, relu=True) == "simt64"
    assert L(1000, 3, 64, sm, group=4) == "simt64" and L(1000, 3, 64, sm, addend=True) == "simt64"
    # SIMT tile width
    assert L(1000, 16, 64, sm) == "simt64" and L(1000, 16, 65, sm) == "simt128"
    # tensor cores: width 128 needs Cout % 128 == 0 and at least one 128-row x 128-column tile per SM
    rows_at = sm * 128
    assert L(rows_at, 64, 128, sm, precision=1) == "tc128"
    assert L(rows_at - 128, 64, 128, sm, precision=1) == "tc64"
    assert L(rows_at // 2, 64, 256, sm, precision=1) == "tc128" and L(rows_at // 2 - 128, 64, 256, sm, precision=1) == "tc64"
    assert L(10 ** 6, 64, 192, sm, precision=1) == "tc64"
    assert L(rows_at, 64, 128, sm, precision=1, group=128) == "tc128+combine"
    assert L(rows_at, 64, 128, sm, precision=1, group=64) == "tc128"
    assert L(4096, 64, 64, sm, precision=1, group=128, single=True) == "tc64+combine+tf32"


def test_layer_dispatch_depends_on_sm_count():
    # 17000 rows = 133 row tiles: width 128 on both SKUs; 16000 rows = 125 tiles: 64 on 132 SMs, 128 on 114
    assert G.layer_path(17000, 256, 128, H100_SXM, precision=1) == "tc128"
    assert G.layer_path(16000, 256, 128, H100_SXM, precision=1) == "tc64"
    assert G.layer_path(16000, 256, 128, H100_PCIE, precision=1) == "tc128"


@pytest.mark.parametrize("prec", [1, 4])
def test_wgrad_dispatch_edges(prec):
    W = G.wgrad_path
    tc = lambda bn: "tc%d" % bn + ("+tf32" if prec == 4 else "")                  # noqa: E731
    assert W(4096, 64, 128, prec) == tc(128) and W(4096, 64, 192, prec) == tc(64) and W(4096, 64, 64, prec) == tc(64)
    assert W(4095, 64, 128, prec) == "simt"                                       # P >= 4096
    assert W(4096, 60, 128, prec) == "simt" and W(4096, 66, 128, prec) == "simt"  # Cout >= 64, Cout % 4 == 0
    assert W(4096, 100, 128, prec) == tc(128)
    assert W(4096, 64, 96, prec) == "simt"                                        # Cin % 64 == 0
    assert W(4096, 64, 128, prec, ldg=65) == "simt" and W(4096, 64, 128, prec, ldg=68) == tc(128)
    assert W(4096, 64, 128, prec, ldx=129) == "simt" and W(4096, 64, 128, prec, ldx=132) == tc(128)
    assert W(4096, 64, 128, prec, gy_aligned=False) == "simt"
    assert W(4096, 64, 128, prec, x_aligned=False) == "simt"
    assert W(4096, 64, 128, prec, affine_aligned=False) == "simt"
    # narrow kernel, reached at every precision when the tensor-core kernel is not eligible
    assert W(4096, 64, 8, prec) == "narrow" and W(4095, 64, 8, prec) == "simt"
    assert W(4096, 64, 9, prec) == "simt" and W(4096, 48, 8, prec) == "simt" and W(4096, 256, 8, prec) == "narrow"
    assert W(4096, 64, 8, prec, ldg=66) == "simt" and W(4096, 64, 8, prec, gy_aligned=False) == "simt"
    assert W(4096, 64, 8, prec, ldx=11, x_aligned=False) == "narrow"
    assert W(4096, 64, 128, 0) == "simt"


@pytest.mark.parametrize("sm", [H100_SXM, H100_PCIE])
def test_wgrad_split_cases(sm):
    for case in G.WGRAD_CASES:
        cid, P, Cout, Cin, kw = case
        if P is None:
            P = G.wgrad_case_P(P, Cout, Cin, kw, sm)
            splits, rows = G.wgrad_simt_split(P, Cout, Cin, sm)
            assert splits > 1
            assert P - (splits - 1) * rows == (1 if kw["split"] == "tail1" else rows)


@pytest.mark.parametrize("kind", ["layer", "wgrad"])
def test_cases_reach_the_kernel_they_were_written_for(kind):
    """The dispatch restatement applied to every GPU case (on the 132-SM H100 SXM the cases were written for)."""
    if kind == "layer":
        for cid, P, Cin, Cout, kw in G.LAYER_CASES:
            got = G.layer_path(P, Cin, Cout, H100_SXM, precision=0 if kw["prec"] == "fp32" else 1,
                               single=kw["prec"] == "tf32", stats=bool(kw.get("stats")), group=kw.get("group", 0),
                               addend=bool(kw.get("add")), affine=kw["pro"].startswith("affine"),
                               relu=kw["pro"] in ("affine_relu", "relu"))
            assert got == kw["path"], (cid, got)
    else:
        for cid, P, Cout, Cin, kw in G.WGRAD_CASES:
            P = G.wgrad_case_P(P, Cout, Cin, kw, H100_SXM)
            got = G.wgrad_path(P, Cout, Cin, kw["prec"], ldg=Cout + kw.get("ldg_pad", 0), ldx=Cin + kw.get("ldx_pad", 0),
                               gy_aligned=kw.get("gy_off", 0) % 4 == 0, x_aligned=kw.get("x_off", 0) % 4 == 0)
            assert got == kw["path"], (cid, got)


def test_layer_tau_covers_round_toward_zero_accumulation():
    """The 3xTF32 layer bound holds, with a 4x margin, for a model of the kernel's arithmetic whose fp32 accumulator
    rounds toward zero, on the operands of the GPU bound test; the dropped lo*lo terms alone are far below it."""
    X, W, b = G.bound_layer_operands(4096, 256, 128)
    ref = G.layer_ref(X, W, b)
    mag = G.err_bound(X, W, 1.0, (np.broadcast_to(b, ref.shape),))
    model = float((np.abs(G.layer_3x_truncating(X, W, b) - ref) / mag).max())
    terms = float((np.abs(G.layer_ref(X, W, b, mode="3x") - ref) / mag).max())
    print("round-toward-zero model %.3e, 3xTF32 terms alone %.3e, tau %.3e" % (model, terms, G.TAU_LAYER))
    assert 4 * model <= G.TAU_LAYER and 16 * terms <= G.TAU_LAYER
