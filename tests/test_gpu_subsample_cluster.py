"""usip_cloud_subsample at every scan length (csrc/pairgen.cu pair_subset_kernel and pair_subset_cluster_kernel).

The numpy restatement of the selection rule (tests/philox_ref.py) is first shown equal to the one-CTA kernel, whose
rows the training and test loaders already rely on; then the cluster kernel, which runs once the longest scan exceeds
pair_max_scan_rows(), is held to the same restatement bit for bit: above the limit, at N = 10240 and 16384, with a
radius mask that leaves at least N valid rows, fewer than N, or none.  A short scan gets the same rows whichever kernel
its batch runs in, and a scan above the documented cap is refused before any launch."""
import numpy as np
import pytest
import torch

from tests import philox_ref as pr
from tests.util_gpu import dev
from usip_b200 import ops
from usip_b200.data.kitti_detector_loader import synthetic_scan

pytestmark = pytest.mark.gpu

SEED, STEP = 0x1234_5678_9ABC, 3


def _scan(seed, n, C=4):
    return synthetic_scan(seed, n, C=max(C, 6))[:, :C].copy()


def _radius_for(n, n_valid):
    """A radius whose disc holds about n_valid of synthetic_scan's rows (x, z uniform in +-40)."""
    return 80.0 * np.sqrt(n_valid / n / np.pi)


def _run(scans, soc, N, n_cand, radius, seed=SEED, step=STEP):
    """usip_cloud_subsample over host scans; clouds read scans[soc[c]] -> host (rows, cand, start, valid)."""
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    out = ops.cloud_subsample(d(np.concatenate(scans)), d(offsets), d(np.asarray(soc, np.int32)),
                              max(len(s) for s in scans), N, n_cand, radius, seed, step)
    return [t.cpu().numpy() for t in out]


def _check(scans, soc, N, n_cand, radius):
    rows, cand, start, valid = _run(scans, soc, N, n_cand, radius)
    for c, s in enumerate(soc):
        ref_rows, ref_valid = pr.subset_rows(scans[s][:, :3], N, SEED, STEP, c, radius)
        ref_cand, ref_start = pr.subset_candidates(N, n_cand, SEED, STEP, c)
        assert valid[c] == ref_valid
        np.testing.assert_array_equal(rows[c], ref_rows)
        np.testing.assert_array_equal(cand[c], ref_cand)
        assert start[c] == ref_start
    return valid


@pytest.mark.parametrize("n", [20480, 57088])
@pytest.mark.parametrize("mask", ["all", "fewer", "none"])
def test_restatement_equals_one_cta_kernel(n, mask):
    assert n <= ops.pair_max_scan_rows()
    N = 10240
    radius = {"all": None, "fewer": _radius_for(n, N // 3), "none": -1.0}[mask]
    scans = [_scan(1, n), _scan(2, n - 77)]
    valid = _check(scans, [0, 1, 1, 0], N, N // 4, radius)
    if mask == "fewer":
        assert 0 < valid.min() and valid.max() < N
    if mask == "none":
        assert (valid == 0).all()


@pytest.mark.parametrize("n", [57089, 200000, 1000003])
@pytest.mark.parametrize("N", [10240, 16384])
@pytest.mark.parametrize("mask", ["at_least_n", "fewer", "none"])
def test_cluster_kernel_equals_restatement(n, N, mask):
    assert n > ops.pair_max_scan_rows()
    # radii from the shorter scan (n // 2 rows): at least N valid in both, or fewer than N in both
    radius = {"at_least_n": _radius_for(n // 2, 2 * N), "fewer": _radius_for(n, N // 3), "none": -1.0}[mask]
    scans = [_scan(10 + n % 97, n), _scan(11, n // 2)]
    valid = _check(scans, [0, 1], N, N // 2, radius)
    if mask == "at_least_n":
        assert valid.min() >= N
    elif mask == "fewer":
        assert 0 < valid.min() and valid.max() < N
    else:
        assert (valid == 0).all()


def test_cluster_kernel_without_radius():
    n, N = 300001, 16384
    valid = _check([_scan(5, n)], [0, 0], N, N // 4, None)
    assert (valid == n).all()


def test_both_kernels_agree_on_a_short_scan():
    short, long_ = _scan(21, 1300), _scan(22, 60000)
    N = 4096
    for radius in (None, 30.0):
        mixed = _run([short, long_], [0, 1], N, N // 4, radius)          # longest scan 60000: cluster kernel
        alone = _run([short], [0, 0], N, N // 4, radius)                 # longest scan 1300: one-CTA kernel
        for a, b in zip(mixed, alone):
            np.testing.assert_array_equal(a[0], b[0])
        ref, _ = pr.subset_rows(short[:, :3], N, SEED, STEP, 0, radius)
        np.testing.assert_array_equal(mixed[0][0], ref)


def test_longest_accepted_scan():
    n, N = ops.SUBSAMPLE_MAX_ROWS, 16384
    scan = np.random.RandomState(3).uniform(-40, 40, (n, 3)).astype(np.float32)
    rows, cand, start, valid = _run([scan], [0, 0], N, N // 4, 20.0)
    for c in range(2):
        ref, ref_valid = pr.subset_rows(scan, N, SEED, STEP, c, 20.0)
        assert valid[c] == ref_valid
        np.testing.assert_array_equal(rows[c], ref)


def test_scan_above_the_cap_is_refused():
    scan = torch.zeros((64, 4), dtype=torch.float32, device=dev())
    offsets = torch.tensor([0, 64], dtype=torch.int64, device=dev())
    soc = torch.zeros(2, dtype=torch.int32, device=dev())
    with pytest.raises(RuntimeError, match="at most 16777216 rows"):
        ops.cloud_subsample(scan, offsets, soc, ops.SUBSAMPLE_MAX_ROWS + 1, 32, 8)
    with pytest.raises(RuntimeError, match="N too large"):
        ops.cloud_subsample(scan, offsets, soc, 64, ops.pair_max_scan_rows() + 1, 8)
