"""Host logic of the indoor registration benchmark (usip_b200.evaluation.indoor_registration): the gt.info, gt.log and
result-log readers, dcm2quat, mrEvaluateRegistrationMy's rules, the all-pairs order, writeLog's filters, the .log
round trip and the refusals -- against tests/indoor_reg_ref.py where a restatement exists.  No GPU."""
import os

import numpy as np
import pytest

from tests import indoor_reg_ref as ir
from usip_b200.evaluation import indoor_registration as idr
from usip_b200.evaluation import indoor_test_loader as itl
from usip_b200.evaluation import registration as reg

GOLDEN_INFO = os.path.join(os.path.dirname(__file__), "golden", "redwood_livingroom1_gt.info")


def _rot(axis, deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    R = np.eye(3)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def _T(R=np.eye(3), t=(0, 0, 0)):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


# ----------------------------------------------------------------------------------------------- readers
def test_read_gt_info_golden_matches_restatement():
    head, info = idr.read_gt_info(GOLDEN_INFO)
    ref = ir.load_info(GOLDEN_INFO)
    assert len(head) == len(ref) == 327
    for e, (x, m) in enumerate(ref):
        assert list(head[e]) == x
        np.testing.assert_array_equal(info[e], m)
    assert list(head[0]) == [0, 1, 57] and info[0, 0, 0] == 3305.0 and info[0, 0, 4] == 10048.00680351
    np.testing.assert_allclose(info, np.swapaxes(info, 1, 2), rtol=1e-9)


def test_gt_info_and_log_order(tmp_path):
    rng = np.random.RandomState(0)
    pairs = [(0, 1), (3, 9), (0, 2), (4, 4)]
    entries = [(a, b, 10, _T(_rot(a % 3, 10 * b), rng.normal(size=3))) for a, b in pairs]
    infos = [(a, b, 10, itl.info_matrix(rng.normal(size=(5, 3)))) for a, b in pairs]
    itl.write_gt_log(str(tmp_path / "gt.log"), entries)
    itl.write_gt_info(str(tmp_path / "gt.info"), infos)
    h1, T = idr.read_gt_log4(str(tmp_path / "gt.log"))
    h2, M = idr.read_gt_info(str(tmp_path / "gt.info"))
    np.testing.assert_array_equal(h1, h2)
    assert [tuple(h[:2]) for h in h1] == pairs and (h1[:, 2] == 10).all()
    np.testing.assert_allclose(T, [e[3] for e in entries], rtol=1e-12)
    np.testing.assert_allclose(M, [e[3] for e in infos], rtol=1e-12)


def test_log_round_trip_matches_restatement(tmp_path):
    rng = np.random.RandomState(1)
    entries = []
    for i, j in [(0, 1), (0, 5), (2, 9)]:
        info = itl.info_matrix(rng.normal(size=(4, 3)))
        info[0, 5] += 1.0                                         # not symmetric: the column order shows
        entries.append((i, j, 12, _T(_rot(1, 5.0), rng.normal(size=3)), int(rng.randint(3, 99)), rng.uniform(), info))
    path = str(tmp_path / "scene.log")
    with open(path, "w") as f:
        for e in entries:
            f.write(idr.format_log_entry(*e))
    got = idr.read_registration_log(path)
    ref = ir.load_log_my(path)
    for e, r in enumerate(ref):
        assert list(got["head"][e]) == r["info"]
        np.testing.assert_array_equal(got["T"][e], r["trans"])
        assert got["inlier_num"][e] == r["inlierNum"] and got["inlier_ratio"][e] == r["inlierRatio"]
        np.testing.assert_array_equal(got["info"][e], r["information"])
        np.testing.assert_allclose(got["info"][e], entries[e][6], atol=1e-10)
        np.testing.assert_allclose(got["T"][e], entries[e][3], atol=1e-10)
    text = open(path).read().splitlines()
    assert text[0] == "0\t 1\t 12\t" and text[5].count("\t") == 1


# ----------------------------------------------------------------------------------------------- the score
def test_dcm2quat_hand_cases():
    np.testing.assert_allclose(idr.dcm2quat(np.eye(3)), [1, 0, 0, 0])
    q = idr.dcm2quat(_rot(2, 90))                                 # about z: the toolbox's sign, -sin(45)
    np.testing.assert_allclose(q, [np.sqrt(0.5), 0, 0, -np.sqrt(0.5)], atol=1e-15)
    q = idr.dcm2quat(_rot(0, 60))
    np.testing.assert_allclose(q, [np.cos(np.radians(30)), -np.sin(np.radians(30)), 0, 0], atol=1e-15)
    assert np.isnan(idr.dcm2quat(np.diag([-1.0, -1.0, 1.0]))[1])  # 180 degrees: q0 = 0, 0 / 0


def _score(result_pairs, result_T, gt_pairs, gt_T, info=None, num=10):
    gt_head = np.array([(a, b, num) for a, b in gt_pairs])
    info = np.broadcast_to(np.eye(6), (len(gt_pairs), 6, 6)) if info is None else info
    res = {"head": np.array([(a, b, num) for a, b in result_pairs]).reshape(-1, 3), "T": np.array(result_T),
           "inlier_num": np.arange(len(result_pairs)) + 10.0, "inlier_ratio": np.linspace(0.1, 0.5, len(result_pairs))}
    got = idr.evaluate_registration(res, gt_head, np.array(gt_T), info)
    ref = ir.evaluate_my([dict(info=list(h), trans=T, inlierNum=n, inlierRatio=r) for h, T, n, r in
                          zip(res["head"], res["T"], res["inlier_num"], res["inlier_ratio"])],
                         [dict(info=list(h), trans=T) for h, T in zip(gt_head, gt_T)], list(info))
    for k in ("recall", "precision", "good", "gt_num", "rs_num", "inlier_num", "inlier_ratio"):
        assert np.isnan(got[k]) and np.isnan(ref[k]) or got[k] == ref[k], k
    return got


def test_score_rules():
    I = np.eye(4)
    gt_pairs = [(0, 1), (0, 2), (3, 7), (4, 6)]
    gt_T = [I, I, _T(t=(1, 0, 0)), I]
    info = np.broadcast_to(np.eye(6), (4, 6, 6)).copy()
    info[1, 1, 1] = 0.04
    t02 = _T(t=(0, 1, 0))                                         # p = 0.04 * 1 / 1 exactly: good
    far = _T(t=(0.3, 0, 0))
    res_pairs = [(0, 1), (0, 2), (3, 7), (4, 6), (5, 9)]          # adjacent (0, 1) ignored; (5, 9) a false positive
    got = _score(res_pairs, [far, t02, _T(t=(1.1, 0, 0)), far, I], gt_pairs, gt_T, info)
    assert got["gt_num"] == 3 and got["rs_num"] == 4 and got["false_pos"] == 1
    assert got["good"] == 2 and got["bad"] == 1 and got["errors"][0] == pytest.approx(0.04, abs=0)
    assert got["recall"] == 2 / 3 and got["precision"] == 2 / 4
    assert got["inlier_num"] == np.mean([11.0, 12.0])
    empty = _score([], np.zeros((0, 4, 4)), gt_pairs, gt_T)
    assert empty["recall"] == 0 and np.isnan(empty["precision"]) and np.isnan(empty["inlier_num"])
    nan_T = _T(np.diag([-1.0, -1.0, 1.0]))                        # p NaN: bad
    assert _score([(0, 2)], [nan_T], gt_pairs, gt_T)["bad"] == 1


def test_score_uses_info_weighting():
    info = np.diag([4.0, 1, 1, 100, 100, 100])[None].repeat(1, 0)
    got = _score([(0, 2)], [_T(_rot(2, 2.0))], [(0, 2)], [np.eye(4)], info)
    q3 = np.sin(np.radians(1.0))
    assert got["errors"][0] == pytest.approx(100 * q3 * q3 / 4, rel=1e-12)


def test_summary_line():
    s = [dict(recall=1.0, precision=0.5, inlier_num=10.0, inlier_ratio=0.25),
         dict(recall=0.5, precision=0.5, inlier_num=13.0, inlier_ratio=0.75)]
    line, m = idr.summary_line(s)
    assert line == "Mean registration recall: 0.750000 precision: 0.500000 inlierNum: 12 inlierRatio: 0.500000"
    s[0]["inlier_num"] = float("nan")
    assert "inlierNum: NaN" in idr.summary_line(s)[0]


# ----------------------------------------------------------------------------------------------- pairs and filters
class _Bare(idr.IndoorRegistration):
    def __init__(self, frames, gt_pairs=()):
        self.scenes = list(frames)
        self.frames_of = frames
        self.gt = {s: (np.array([(a, b, len(f)) for a, b in gt_pairs]).reshape(-1, 3), None, None)
                   for s, f in frames.items()}
        self.overlap_calls = []

    def _overlap(self, scene, fp, Rt, candidate):
        self.overlap_calls.append(candidate.copy())
        return np.array([0.23, 0.2300001, 0.5, 0.9])[:candidate.sum()]


def test_all_pairs_order():
    ev = _Bare({"a": [0, 1, 2, 3], "b": [0, 2, 10]}, gt_pairs=[(2, 3), (0, 1)])
    assert ev.scene_pairs("a").tolist() == [[0, 1], [0, 2], [0, 3], [1, 2], [1, 3], [2, 3]]
    assert ev.scene_pairs("b").tolist() == [[0, 2], [0, 10], [2, 10]]
    assert ev.scene_pairs("a", "gt").tolist() == [[2, 3], [0, 1]]
    with pytest.raises(ValueError):
        ev.scene_pairs("a", "some")
    assert len(_Bare({"s": list(range(57))}).scene_pairs("s")) == 57 * 56 // 2


def test_writelog_filters_are_strict():
    ev = _Bare({"s": [0, 1, 2, 3, 4]})
    fp = np.array([[0, 2], [0, 3], [1, 3], [1, 4], [2, 4]])
    n_m = np.array([[1000], [1000], [1000], [1000], [0]], np.int32)
    r = {"n_matches": n_m, "Rt": np.zeros((5, 1, 1, 3, 4)), "status": np.array([0, 0, 0, 0, 1]).reshape(5, 1, 1),
         "n_inliers": np.array([25, 26, 30, 40, 9]).reshape(5, 1, 1), "info": np.zeros((5, 1, 1, 6, 6)),
         "n_info": np.zeros((5, 1, 1), np.int32)}
    r["Rt"][..., :3] = np.eye(3)
    out = ev._finish("s", fp, r, 1, 1, 0.23)
    # 25 / 1000 = 0.025 is not above 0.025; the rest run the overlap test, 0.23 itself is not above 0.23
    assert ev.overlap_calls[0][:, 0, 0].tolist() == [False, True, True, True, False]
    assert out["accepted"][:, 0, 0].tolist() == [False, False, True, True, False]
    assert out["n_inliers"][4, 0, 0] == 0 and np.array_equal(out["Rt"][4, 0, 0], np.eye(4))
    lite = ev._finish("s", fp, r, 1, 1, None)
    assert len(ev.overlap_calls) == 1 and lite["accepted"][:, 0, 0].tolist() == [False, True, True, True, False]


# ----------------------------------------------------------------------------------------------- refusals
def test_refusals(tmp_path):
    ev = _Bare({"s": [0, 1]})
    ev.xyz = None
    with pytest.raises(RuntimeError):
        ev.score([8], [1000])
    with pytest.raises(ValueError):
        ev.score([8, 4], [1000])
    with pytest.raises(ValueError):
        ev.score([8], [30000, 1000])
    with pytest.raises(ValueError):
        ev.score([2048], [1000])
    with pytest.raises(RuntimeError):
        ev.result = None
        ev.write_registration_logs(str(tmp_path), 8, 1000)
    bad = tmp_path / "bad.info"
    bad.write_text("0 1 5\n1 2 3\n")
    with pytest.raises(ValueError):
        idr.read_gt_info(str(bad))
    with pytest.raises(SystemExit):
        idr.main(["redwood", "--root", str(tmp_path)])                    # no --gt-root
    with pytest.raises(SystemExit):
        idr.main(["3dmatch", "--root", str(tmp_path)])                    # neither a tree nor a model


def test_score_logs_cli(tmp_path, capsys):
    scenes = [s for s, _ in itl.REDWOOD_SCENES]
    for s in scenes:
        d = tmp_path / "gt" / "original" / ("%s-evaluation" % s)
        itl.write_gt_log(str(d / "gt.log"), [(0, 2, 5, np.eye(4)), (1, 4, 5, _T(t=(1, 0, 0)))])
        itl.write_gt_info(str(d / "gt.info"), [(0, 2, 5, np.eye(6)), (1, 4, 5, np.eye(6))])
    logs = tmp_path / "logs"
    logs.mkdir()
    (logs / "livingroom1.log").write_text(idr.format_log_entry(0, 2, 5, np.eye(4), 30, 0.5, np.eye(6)))
    sc = idr.main(["redwood", "--gt-root", str(tmp_path / "gt"), "--score-logs", str(logs)])
    assert sc["livingroom1"]["recall"] == 0.5 and sc["livingroom1"]["precision"] == 1.0
    assert sc["office1"]["recall"] == 0 and np.isnan(sc["office1"]["precision"])
    assert "Mean registration recall: 0.125000 precision: NaN" in capsys.readouterr().out


def test_descriptor_opt_indoor():
    o = reg.descriptor_opt("redwood")
    assert (o.ball_radius, o.ball_nsamples, o.descriptor_len, o.sigma_max) == (0.75, 448, 128, 0.5)
    assert reg.descriptor_opt("3dmatch", ball_nsamples=64).ball_nsamples == 64
    assert reg.descriptor_opt("kitti").ball_nsamples == 64
