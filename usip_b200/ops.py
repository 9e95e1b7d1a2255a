"""Thin torch-tensor wrappers over the C ABI (include/usip_b200.h).  PyTorch is used for device
memory and streams only; every computation below happens in libusip_b200.so.  All functions launch on
torch's current CUDA stream and never synchronise."""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import LayerDesc, check

i32 = torch.int32
f32 = torch.float32


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _req(t, dtype, name):
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor/variable" % name)       # index_max.cpp:119-121
    if not t.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)
    if t.dtype != dtype:
        raise RuntimeError("%s: expected dtype %s, got %s" % (name, dtype, t.dtype))


def stat_slots(P, Cout, precision=0, group=0, want_group=False):
    """Rows of the [slots, 2, Cout] BN-statistic partial buffer usip_layer_fwd fills for this layer shape."""
    d = _lib.LayerDesc()
    d.P, d.Cout, d.precision, d.group = int(P), int(Cout), int(precision), int(group)
    d.gmax = 1 if want_group else None          # only tested for NULL-ness by the query
    return _lib.load().usip_layer_stat_slots(ctypes.byref(d))


# ----------------------------------------------------------------------------- reference operators
def index_max(data, index, K):
    """(B,C,N) f32, (B,N) i32 -> (B,C,K) i32.  index_max.forward_cuda_shared_mem semantics."""
    _req(data, f32, "data"); _req(index, i32, "index")
    B, C, N = data.shape
    out = torch.empty((B, C, int(K)), dtype=i32, device=data.device)
    scratch = None
    if K * 12 > 200 * 1024:
        scratch = torch.empty((B * C * K,), dtype=torch.int64, device=data.device)
    with torch.cuda.device(data.device):
        check(_lib.load().usip_index_max_f32(_p(data), _p(index), _p(out), _p(scratch), B, C, N, int(K), _stream()),
              "usip_index_max_f32")
    return out


def ball_query_dist(dist, radius, K):
    _req(dist, f32, "node_to_point_dist")
    B, M, N = dist.shape
    out = torch.empty((B, M, int(K)), dtype=i32, device=dist.device)
    with torch.cuda.device(dist.device):
        check(_lib.load().usip_ball_query_dist_f32(_p(dist), float(radius), _p(out), B, M, N, int(K), _stream()),
              "usip_ball_query_dist_f32")
    return out


_BG_SCRATCH = {}


def _ball_group_scratch(lib, device, B, S, N, M, K):
    """Persistent scratch of the bucket-grid ball query, one per (device, stream, batch): its counter region is cleared once
    here and left cleared by every call (include/usip_b200.h), so the hot path launches no memset."""
    stream = torch.cuda.current_stream()
    key = (device.index, stream.cuda_stream, B)
    ent = _BG_SCRATCH.get(key)
    if ent is None:
        nbytes = int(lib.usip_ball_group_scratch_bytes(B, S, N, M, K))
        buf = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=device)
        check(lib.usip_ball_group_scratch_init(_p(buf), nbytes, B, _stream()), "usip_ball_group_scratch_init")
        _lib.LAUNCHES[0] -= 1                      # a memset, not one of our kernels
        ent = _BG_SCRATCH[key] = (buf, nbytes)
    return ent


def ball_group(xyz, feat, centers, radius, K, want_group=True, rows_ld=0):
    """Fused distance + ball query + gather + decentre.  Returns (idx (B,M,K) i32, group (B,3+S,M,K) f32)."""
    _req(xyz, f32, "xyz"); _req(centers, f32, "centers")
    B, _, N = xyz.shape
    M = centers.shape[2]
    S = 0 if feat is None else feat.shape[1]
    if S:
        _req(feat, f32, "feat")
    lib = _lib.load()
    idx = torch.empty((B, M, int(K)), dtype=i32, device=xyz.device)
    grp = torch.empty((B, 3 + S, M, int(K)), dtype=f32, device=xyz.device) if want_group else None
    rows = torch.empty((B * M * int(K), rows_ld), dtype=f32, device=xyz.device) if rows_ld else None
    with torch.cuda.device(xyz.device):
        scratch, nbytes = _ball_group_scratch(lib, xyz.device, B, S, N, M, int(K))
        check(lib.usip_ball_group_f32(_p(xyz), _p(feat) if S else None, _p(centers), float(radius), _p(idx), _p(grp),
                                      _p(rows), rows_ld, _p(scratch), int(nbytes), B, S, N, M, int(K), _stream()),
              "usip_ball_group_f32")
    if rows_ld:
        return idx, grp, rows
    return idx, grp


def knn_group(xyz, feat, centers, K, want_group=True, rows_ld=0):
    """K nearest points of every centre + gather + decentre (RPN_Detector_KNN front end, networks.py:556-565).
    Returns (idx (B,M,K) i32 ascending, group (B,3+S,M,K) f32 or None[, rows [B*M*K, rows_ld]])."""
    _req(xyz, f32, "xyz"); _req(centers, f32, "centers")
    B, _, N = xyz.shape
    M = centers.shape[2]
    S = 0 if feat is None else feat.shape[1]
    if S:
        _req(feat, f32, "feat")
    idx = torch.empty((B, M, int(K)), dtype=i32, device=xyz.device)
    grp = torch.empty((B, 3 + S, M, int(K)), dtype=f32, device=xyz.device) if want_group else None
    rows = torch.empty((B * M * int(K), rows_ld), dtype=f32, device=xyz.device) if rows_ld else None
    with torch.cuda.device(xyz.device):
        check(_lib.load().usip_knn_group_f32(_p(xyz), _p(feat) if S else None, _p(centers), _p(idx), _p(grp), _p(rows), rows_ld,
                                             B, S, N, M, int(K), _stream()), "usip_knn_group_f32")
    if rows_ld:
        return idx, grp, rows
    return idx, grp


def fps(pts, start, k, want_nodes=True):
    """Farthest point sampling.  pts (B,Ns,3) f32, start (B,) i32 -> (idx (B,k) i32, nodes (B,3,k) f32 or None)."""
    _req(pts, f32, "pts"); _req(start, i32, "start")
    B, Ns, _ = pts.shape
    idx = torch.empty((B, int(k)), dtype=i32, device=pts.device)
    nodes = torch.empty((B, 3, int(k)), dtype=f32, device=pts.device) if want_nodes else None
    with torch.cuda.device(pts.device):
        check(_lib.load().usip_fps_f32(_p(pts), _p(start), _p(idx), _p(nodes), B, Ns, int(k), _stream()), "usip_fps_f32")
    return idx, nodes


def fps_f64(pts, start, k, want_nodes=False):
    """fps on float64 points: pts (B,Ns,3) f64, start (B,) i32 -> (idx (B,k) i32, nodes (B,3,k) f32 casts or None)."""
    _req(pts, torch.float64, "pts"); _req(start, i32, "start")
    B, Ns, _ = pts.shape
    idx = torch.empty((B, int(k)), dtype=i32, device=pts.device)
    nodes = torch.empty((B, 3, int(k)), dtype=f32, device=pts.device) if want_nodes else None
    with torch.cuda.device(pts.device):
        check(_lib.load().usip_fps_f64(_p(pts), _p(start), _p(idx), _p(nodes), B, Ns, int(k), _stream()), "usip_fps_f64")
    return idx, nodes


# ----------------------------------------------------------------------------- training pairs (csrc/pairgen.cu)
PAIR_TRAIN, PAIR_ROT_HORIZONTAL, PAIR_ROT_3D, PAIR_ROT_PERTURBATION, PAIR_TRANSLATION = 1, 2, 4, 8, 16
PAIR_ENU_TO_CAM, PAIR_HEIGHT_SCALE = 32, 64      # Oxford: camera frame first; detector height scale = params[:, 44]
PAIR_PARAM_STRIDE = 48                           # detector: doubles per pair
PAIR_AUGMENT_SLOT = 45                           # indoor_pair_augment: params[:, 45] != 0 augments the pair
SUBSAMPLE_MAX_ROWS = 1 << 24                     # cloud_subsample: the longest scan (USIP_SUBSAMPLE_MAX_ROWS)
DESC_PARAM_STRIDE = 32                           # descriptor: doubles per cloud
SCENENN_KIND_NONE, SCENENN_KIND_ROT, SCENENN_KIND_FULL = 0, 1, 2   # scenenn_desc_pair_augment: params[:, 45]


def pair_max_scan_rows():
    return _lib.load().usip_pair_max_scan_rows()


def _req_scans(scans, offsets, scan_of_cloud):
    _req(scans, f32, "scans"); _req(offsets, torch.int64, "offsets"); _req(scan_of_cloud, i32, "scan_of_cloud")
    if scans.dim() != 2 or scans.shape[1] < 3:
        raise ValueError("scans must be [T, C] with C >= 3")
    if scan_of_cloud.dim() != 1 or scan_of_cloud.shape[0] == 0 or scan_of_cloud.shape[0] % 2:
        raise ValueError("scan_of_cloud must name the scans of both clouds of every pair: (2B,) with B >= 1")


def _req_jitter(jit_pc, jit_sn, jit_node):
    for name, j in (("jit_pc", jit_pc), ("jit_sn", jit_sn), ("jit_node", jit_node)):
        if j is not None:
            _req(j, torch.float64, name)


def cloud_subsample(scans, offsets, scan_of_cloud, max_rows, N, n_cand, radius=None, seed=0, step=0):
    """Device-mode subsets of 2B clouds.  scans [T, C] f32, offsets (n_scans+1,) i64, scan_of_cloud (2B,) i32 the scan
    of every cloud -> rows (2B, N) i32, cand (2B, n_cand) i32, start (2B,) i32, valid (2B,) i32 (points inside the
    radius).  max_rows (the longest scan) may be up to SUBSAMPLE_MAX_ROWS; scans longer than pair_max_scan_rows() run
    in the cluster kernel, which selects the same rows.  N <= pair_max_scan_rows()."""
    _req_scans(scans, offsets, scan_of_cloud)
    B, dev = scan_of_cloud.shape[0] // 2, scans.device
    rows = torch.empty((2 * B, int(N)), dtype=i32, device=dev)
    cand = torch.empty((2 * B, int(n_cand)), dtype=i32, device=dev)
    start = torch.empty((2 * B,), dtype=i32, device=dev)
    valid = torch.empty((2 * B,), dtype=i32, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().usip_cloud_subsample(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), int(max_rows), B, int(N), int(n_cand),
            int(radius is not None), float(radius if radius is not None else 0.0), int(seed) & (2 ** 64 - 1),
            int(step) & (2 ** 64 - 1), _p(rows), _p(cand), _p(start), _p(valid), _stream()), "usip_cloud_subsample")
    return rows, cand, start, valid


def cloud_gather_candidates(scans, offsets, scan_of_cloud, rows, cand, z_scale=None):
    """FPS input: (2B, n_cand, 3) f32 xyz of rows[c, cand[c, j]] of scan scan_of_cloud[c].  z_scale (2B,) f32 or
    None: z becomes fl32(z * z_scale[c]) (the Oxford detector's height scaling)."""
    _req_scans(scans, offsets, scan_of_cloud); _req(rows, i32, "rows"); _req(cand, i32, "cand")
    B, N, n_cand = scan_of_cloud.shape[0] // 2, rows.shape[1], cand.shape[1]
    pts = torch.empty((2 * B, n_cand, 3), dtype=f32, device=scans.device)
    lib = _lib.load()
    with torch.cuda.device(scans.device):
        if z_scale is None:
            check(lib.usip_cloud_gather_candidates(_p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows),
                                                   _p(cand), _p(pts), B, N, n_cand, _stream()),
                  "usip_cloud_gather_candidates")
        else:
            _req(z_scale, f32, "z_scale")
            if tuple(z_scale.shape) != (2 * B,):
                raise ValueError("z_scale must be (%d,), one factor per cloud; got %s" % (2 * B, tuple(z_scale.shape)))
            check(lib.usip_cloud_gather_candidates_zscaled(_p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud),
                                                           _p(rows), _p(cand), _p(z_scale), _p(pts), B, N, n_cand,
                                                           _stream()), "usip_cloud_gather_candidates_zscaled")
    return pts


def _req_icp(icp, B):
    _req(icp, torch.float64, "icp")
    if tuple(icp.shape) != (B, 4, 4):
        raise ValueError("icp must be (%d, 4, 4), one matrix per pair; got %s" % (B, tuple(icp.shape)))


def cloud_gather_candidates_icp_f64(scans, offsets, scan_of_cloud, rows, cand, icp):
    """SceneNN descriptor FPS input: (2B, n_cand, 3) f64 xyz of rows[c, cand[c, j]]; the anchor's (c even) mapped by
    hom2cart(icp[c // 2] @ [x y z 1]) in the summation order of include/usip_b200.h, the positive's exact."""
    _req_scans(scans, offsets, scan_of_cloud); _req(rows, i32, "rows"); _req(cand, i32, "cand")
    B, N, n_cand = scan_of_cloud.shape[0] // 2, rows.shape[1], cand.shape[1]
    _req_icp(icp, B)
    pts = torch.empty((2 * B, n_cand, 3), dtype=torch.float64, device=scans.device)
    with torch.cuda.device(scans.device):
        check(_lib.load().usip_cloud_gather_candidates_icp_f64(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows), _p(cand), _p(icp), _p(pts), B, N,
            n_cand, _stream()), "usip_cloud_gather_candidates_icp_f64")
    return pts


def scenenn_desc_pair_augment(scans, offsets, scan_of_cloud, rows, icp, cand_pts, node_idx, params, S, flags):
    """SceneNN descriptor pairs -> (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node, R (B,3,3), scale (B,),
    shift (B,3,1)), all f32.  icp (B,4,4) f64, cand_pts (2B, n_cand, 3) f64 (cloud_gather_candidates_icp_f64), node_idx
    (2B, M) i32 (fps_f64), params (B, 48) f64 with the pair's augmentation kind in params[:, PAIR_AUGMENT_SLOT]
    (SCENENN_KIND_*).  No jitter: the reference loader draws it but never applies it."""
    _req_scans(scans, offsets, scan_of_cloud); _req(rows, i32, "rows"); _req(node_idx, i32, "node_idx")
    _req(cand_pts, torch.float64, "cand_pts"); _req(params, torch.float64, "params")
    B, N, M, dev = scan_of_cloud.shape[0] // 2, rows.shape[1], node_idx.shape[1], scans.device
    _req_icp(icp, B)
    e = lambda *s: torch.empty(s, dtype=f32, device=dev)
    out = (e(B, 3, N), e(B, S, N), e(B, 3, M), e(B, 3, N), e(B, S, N), e(B, 3, M), e(B, 3, 3), e(B), e(B, 3, 1))
    with torch.cuda.device(dev):
        check(_lib.load().usip_scenenn_desc_pair_augment(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows), _p(icp), _p(cand_pts), _p(node_idx),
            _p(params), int(flags), int(S), B, N, M, cand_pts.shape[1], *[_p(t) for t in out], _stream()),
            "usip_scenenn_desc_pair_augment")
    return out


def scale_channel_(t, k, factor):
    """In place: t[:, k, :] *= factor for t (B, C, L) f32 CUDA, in fp32 as torch multiplies a float32 tensor by a
    Python float.  Returns t."""
    _req(t, f32, "t")
    if t.dim() != 3 or not 0 <= int(k) < t.shape[1]:
        raise ValueError("t must be (B, C, L) with 0 <= k < C")
    B, C, L = t.shape
    if t.numel() == 0:
        return t
    with torch.cuda.device(t.device):
        check(_lib.load().usip_scale_channel_f32(_p(t), B, C, L, int(k), float(factor), _stream()),
              "usip_scale_channel_f32")
    return t


def pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, S, flags, seed=0, step=0, jit_pc=None, jit_sn=None,
                 jit_node=None):
    """Detector augmentation + dst transform -> the nine ModelDetector.set_input tensors (src_pc, src_sn, src_node,
    dst_pc, dst_sn, dst_node, R, scale, shift).  params (B, 48) f64 on the device (layout in include/usip_b200.h); jitter
    arrays f64 or None (drawn on the device from (seed, step))."""
    _req_scans(scans, offsets, scan_of_cloud); _req(rows, i32, "rows"); _req(nodes, f32, "nodes")
    _req(params, torch.float64, "params"); _req_jitter(jit_pc, jit_sn, jit_node)
    B, N, M, dev = scan_of_cloud.shape[0] // 2, rows.shape[1], nodes.shape[2], scans.device
    e = lambda *s: torch.empty(s, dtype=f32, device=dev)
    out = (e(B, 3, N), e(B, S, N), e(B, 3, M), e(B, 3, N), e(B, S, N), e(B, 3, M), e(B, 3, 3), e(B), e(B, 3, 1))
    with torch.cuda.device(dev):
        check(_lib.load().usip_pair_augment(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows), _p(nodes), _p(params), _p(jit_pc),
            _p(jit_sn), _p(jit_node), int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1), int(flags), int(S), B, N, M,
            *[_p(t) for t in out], _stream()), "usip_pair_augment")
    return out


def indoor_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, S, flags, seed=0, step=0, jit_pc=None,
                        jit_sn=None, jit_node=None):
    """3DMatch / SceneNN detector augmentation + dst transform -> the nine ModelDetector.set_input tensors, as
    pair_augment but with the indoor jitter laws (sigma 0.01, clip 0.02 for pc, sn and nodes), sn = scan columns 3:3+S
    for every S, and a per-pair switch: with PAIR_TRAIN, pair b is augmented only when params[b, PAIR_AUGMENT_SLOT] != 0.
    Jitter arrays per cloud, (2B, N, 3), (2B, N, S), (2B, M, 3) f64, or None (drawn on the device from (seed, step))."""
    _req_scans(scans, offsets, scan_of_cloud); _req(rows, i32, "rows"); _req(nodes, f32, "nodes")
    _req(params, torch.float64, "params"); _req_jitter(jit_pc, jit_sn, jit_node)
    B, N, M, dev = scan_of_cloud.shape[0] // 2, rows.shape[1], nodes.shape[2], scans.device
    e = lambda *s: torch.empty(s, dtype=f32, device=dev)
    out = (e(B, 3, N), e(B, S, N), e(B, 3, M), e(B, 3, N), e(B, S, N), e(B, 3, M), e(B, 3, 3), e(B), e(B, 3, 1))
    with torch.cuda.device(dev):
        check(_lib.load().usip_indoor_pair_augment(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows), _p(nodes), _p(params), _p(jit_pc),
            _p(jit_sn), _p(jit_node), int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1), int(flags), int(S), B, N, M,
            *[_p(t) for t in out], _stream()), "usip_indoor_pair_augment")
    return out


def modelnet_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, flags, seed=0, step=0, jit_pc=None,
                          jit_sn=None, jit_node=None):
    """ModelNet detector augmentation + dst transform -> the nine ModelDetector.set_input tensors, sn = scan columns
    3:6.  params (B, 48) f64 on the device (layout in include/usip_b200.h); jitter arrays f64 PER PAIR -- jit_pc and
    jit_sn (B, N, 3), jit_node (B, M, 3), shared by the pair's two clouds -- or None (drawn on the device from
    (seed, step))."""
    _req_scans(scans, offsets, scan_of_cloud); _req(rows, i32, "rows"); _req(nodes, f32, "nodes")
    _req(params, torch.float64, "params"); _req_jitter(jit_pc, jit_sn, jit_node)
    B, N, M, dev = scan_of_cloud.shape[0] // 2, rows.shape[1], nodes.shape[2], scans.device
    for name, j, n in (("jit_pc", jit_pc, N), ("jit_sn", jit_sn, N), ("jit_node", jit_node, M)):
        if j is not None and tuple(j.shape) != (B, n, 3):
            raise ValueError("%s must be (%d, %d, 3), one array per pair; got %s" % (name, B, n, tuple(j.shape)))
    e = lambda *s: torch.empty(s, dtype=f32, device=dev)
    out = (e(B, 3, N), e(B, 3, N), e(B, 3, M), e(B, 3, N), e(B, 3, N), e(B, 3, M), e(B, 3, 3), e(B), e(B, 3, 1))
    with torch.cuda.device(dev):
        check(_lib.load().usip_modelnet_pair_augment(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows), _p(nodes), _p(params), _p(jit_pc),
            _p(jit_sn), _p(jit_node), int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1), int(flags), 3, B, N, M,
            *[_p(t) for t in out], _stream()), "usip_modelnet_pair_augment")
    return out


def desc_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, S, flags, seed=0, step=0, jit_pc=None,
                      jit_sn=None, jit_node=None):
    """Descriptor augmentation -> (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node).  params (2B, 32) f64 per cloud
    on the device (layout in include/usip_b200.h); jitter arrays f64 or None (drawn on the device from (seed, step))."""
    _req_scans(scans, offsets, scan_of_cloud); _req(rows, i32, "rows"); _req(nodes, f32, "nodes")
    _req(params, torch.float64, "params"); _req_jitter(jit_pc, jit_sn, jit_node)
    B, N, M, dev = scan_of_cloud.shape[0] // 2, rows.shape[1], nodes.shape[2], scans.device
    e = lambda *s: torch.empty(s, dtype=f32, device=dev)
    out = (e(B, 3, N), e(B, S, N), e(B, 3, M), e(B, 3, N), e(B, S, N), e(B, 3, M))
    with torch.cuda.device(dev):
        check(_lib.load().usip_desc_pair_augment(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows), _p(nodes), _p(params), _p(jit_pc),
            _p(jit_sn), _p(jit_node), int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1), int(flags), int(S), B, N, M,
            *[_p(t) for t in out], _stream()), "usip_desc_pair_augment")
    return out


def test_cloud_gather(scans, offsets, scan_of_cloud, rows, nodes, S, flags=0, noise_sigma=0.0, noise=None, seed=0,
                      step=0):
    """Test-set clouds (no augmentation, no pair) -> (pc (B,3,N), sn (B,S,N), node (B,3,M)) f32, B = len(scan_of_cloud).
    flags: 0 or PAIR_ENU_TO_CAM.  noise_sigma != 0 adds fl32(n * sigma) to pc, n = noise (B,3,N) f32 or, when None,
    Philox N(0, 1) drawn from (seed, step)."""
    _req(scans, f32, "scans"); _req(offsets, torch.int64, "offsets"); _req(scan_of_cloud, i32, "scan_of_cloud")
    _req(rows, i32, "rows"); _req(nodes, f32, "nodes")
    B, N, M, dev = scan_of_cloud.shape[0], rows.shape[1], nodes.shape[2], scans.device
    if scans.dim() != 2 or rows.shape[0] != B or tuple(nodes.shape[:2]) != (B, 3):
        raise ValueError("scans [T, C], rows (B, N), nodes (B, 3, M) with B = len(scan_of_cloud)")
    if noise is not None:
        _req(noise, f32, "noise")
        if tuple(noise.shape) != (B, 3, N):
            raise ValueError("noise must be (%d, 3, %d); got %s" % (B, N, tuple(noise.shape)))
    e = lambda *s: torch.empty(s, dtype=f32, device=dev)
    out = (e(B, 3, N), e(B, int(S), N), e(B, 3, M))
    with torch.cuda.device(dev):
        check(_lib.load().usip_test_cloud_gather(
            _p(scans), scans.shape[1], _p(offsets), _p(scan_of_cloud), _p(rows), _p(nodes), _p(noise),
            float(noise_sigma), int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1), int(flags), int(S), B, N, M,
            *[_p(t) for t in out], _stream()), "usip_test_cloud_gather")
    return out


def repeatability(keypoints, order, count, pairs, frames, ks, radius):
    """eval_rep.m's inlier counts for every K at once (include/usip_b200.h usip_repeatability_f64).  keypoints
    (S,3,M) f32, order (S,M) i32, count (S,) i32, pairs (P,2) i32, frames (P,3,3,4) f64 (F_a, F_p, T_gt), all CUDA;
    ks ascending ints (host) -> (inliers (P,nK) i32, n_anc (P,nK) i32)."""
    _req(keypoints, f32, "keypoints"); _req(order, i32, "order"); _req(count, i32, "count")
    _req(pairs, i32, "pairs"); _req(frames, torch.float64, "frames")
    S, _, M = keypoints.shape
    P = pairs.shape[0]
    if tuple(order.shape) != (S, M) or tuple(count.shape) != (S,):
        raise ValueError("order must be (%d, %d) and count (%d,)" % (S, M, S))
    if pairs.dim() != 2 or pairs.shape[1] != 2 or tuple(frames.shape) != (P, 3, 3, 4):
        raise ValueError("pairs must be (P, 2) and frames (P, 3, 3, 4)")
    ks_h = (ctypes.c_int32 * len(ks))(*[int(k) for k in ks])
    inl = torch.empty((P, len(ks)), dtype=i32, device=keypoints.device)
    n_anc = torch.empty((P, len(ks)), dtype=i32, device=keypoints.device)
    with torch.cuda.device(keypoints.device):
        check(_lib.load().usip_repeatability_f64(
            _p(keypoints), _p(order), _p(count), S, M, _p(pairs), _p(frames), P, ks_h, len(ks), float(radius),
            _p(inl), _p(n_anc), _stream()), "usip_repeatability_f64")
    return inl, n_anc


def desc_match(desc, count, pairs, ks, k):
    """Descriptor matches of evaluate_kitti.m (k == 1) / evaluate_oxford.m (k in 2..8) for every pair and K at once
    (include/usip_b200.h usip_desc_match_f64).  desc (S,L,D) f32, count (S,) i32, pairs (P,2) i32, all CUDA; ks
    ascending ints (host) -> (matches (P,nK,cap,2) i32, n_matches (P,nK) i32), cap = L for k == 1, 2*k*L otherwise."""
    _req(desc, f32, "desc"); _req(count, i32, "count"); _req(pairs, i32, "pairs")
    S, L, D = desc.shape
    P = pairs.shape[0]
    if tuple(count.shape) != (S,) or pairs.dim() != 2 or pairs.shape[1] != 2:
        raise ValueError("count must be (%d,) and pairs (P, 2)" % S)
    ks_h = (ctypes.c_int32 * len(ks))(*[int(v) for v in ks])
    cap = (L if int(k) == 1 else 2 * int(k) * L) if 1 <= int(k) <= 8 else 1      # the C call refuses a bad k
    matches = torch.empty((P, len(ks), cap, 2), dtype=i32, device=desc.device)
    n = torch.empty((P, len(ks)), dtype=i32, device=desc.device)
    with torch.cuda.device(desc.device):
        check(_lib.load().usip_desc_match_f64(_p(desc), _p(count), S, L, D, _p(pairs), P, ks_h, len(ks), int(k),
                                              _p(matches), _p(n), _stream()), "usip_desc_match_f64")
    return matches, n


def ransac_rt(xyz, count, pairs, frames, matches, n_matches, trials, threshold=1.0, seed=0, uniforms=None):
    """ransacfitRt.m for every pair, K and trial budget at once (include/usip_b200.h usip_ransac_rt_f64).  xyz (S,L,3)
    f32, count (S,) i32, pairs (P,2) i32, frames (P,3,3,4) f64, matches / n_matches from desc_match, all CUDA; trials
    ascending ints (host); uniforms None (Philox from seed) or (trials[-1] + 1, 3) f64 CUDA -> dict of Rt
    (P,nK,nT,3,4) f64 and n_inliers, trialcount, best_trial, status (P,nK,nT) i32."""
    _req(xyz, f32, "xyz"); _req(count, i32, "count"); _req(pairs, i32, "pairs"); _req(frames, torch.float64, "frames")
    _req(matches, i32, "matches"); _req(n_matches, i32, "n_matches")
    S, L, _ = xyz.shape
    P, nK, cap = matches.shape[0], matches.shape[1], matches.shape[2]
    if tuple(xyz.shape) != (S, L, 3) or tuple(count.shape) != (S,) or tuple(pairs.shape) != (P, 2):
        raise ValueError("xyz must be (S, L, 3), count (S,) and pairs (P, 2)")
    if tuple(frames.shape) != (P, 3, 3, 4) or tuple(matches.shape) != (P, nK, cap, 2) or \
            tuple(n_matches.shape) != (P, nK):
        raise ValueError("frames must be (P, 3, 3, 4), matches (P, nK, cap, 2) and n_matches (P, nK)")
    trials = [int(t) for t in trials]
    if uniforms is not None:
        _req(uniforms, torch.float64, "uniforms")
        if not trials or tuple(uniforms.shape) != (max(trials) + 1, 3):
            raise ValueError("uniforms must be (max(trials) + 1, 3)")
    t_h = (ctypes.c_int32 * len(trials))(*trials)
    nT, dev = len(trials), xyz.device
    Rt = torch.empty((P, nK, nT, 3, 4), dtype=torch.float64, device=dev)
    e = lambda: torch.empty((P, nK, nT), dtype=i32, device=dev)
    out = {"Rt": Rt, "n_inliers": e(), "trialcount": e(), "best_trial": e(), "status": e()}
    with torch.cuda.device(dev):
        check(_lib.load().usip_ransac_rt_f64(
            _p(xyz), _p(count), S, L, _p(pairs), _p(frames), P, nK, _p(matches), _p(n_matches), cap, t_h, nT,
            float(threshold), int(seed) & (2 ** 64 - 1), _p(uniforms), _p(Rt), _p(out["n_inliers"]),
            _p(out["trialcount"]), _p(out["best_trial"]), _p(out["status"]), _stream()), "usip_ransac_rt_f64")
    return out


def ransac_info(xyz, count, pairs, frames, matches, n_matches, trials, best_trial, status, threshold=1.0, seed=0,
                uniforms=None):
    """register2Fragments.m's information matrix of ransac_rt's best models (include/usip_b200.h usip_ransac_info_f64):
    the arguments of ransac_rt, plus its best_trial and status (P,nK,nT) i32 CUDA -> (info (P,nK,nT,6,6) f64, n_info
    (P,nK,nT) i32)."""
    _req(xyz, f32, "xyz"); _req(count, i32, "count"); _req(pairs, i32, "pairs"); _req(frames, torch.float64, "frames")
    _req(matches, i32, "matches"); _req(n_matches, i32, "n_matches")
    _req(best_trial, i32, "best_trial"); _req(status, i32, "status")
    S, L, _ = xyz.shape
    P, nK, cap = matches.shape[0], matches.shape[1], matches.shape[2]
    trials = [int(t) for t in trials]
    nT, dev = len(trials), xyz.device
    if tuple(xyz.shape) != (S, L, 3) or tuple(count.shape) != (S,) or tuple(pairs.shape) != (P, 2):
        raise ValueError("xyz must be (S, L, 3), count (S,) and pairs (P, 2)")
    if tuple(frames.shape) != (P, 3, 3, 4) or tuple(matches.shape) != (P, nK, cap, 2) or \
            tuple(n_matches.shape) != (P, nK):
        raise ValueError("frames must be (P, 3, 3, 4), matches (P, nK, cap, 2) and n_matches (P, nK)")
    if tuple(best_trial.shape) != (P, nK, nT) or tuple(status.shape) != (P, nK, nT):
        raise ValueError("best_trial and status must be (P, nK, nT)")
    if uniforms is not None:
        _req(uniforms, torch.float64, "uniforms")
        if not trials or tuple(uniforms.shape) != (max(trials) + 1, 3):
            raise ValueError("uniforms must be (max(trials) + 1, 3)")
    t_h = (ctypes.c_int32 * nT)(*trials)
    info = torch.empty((P, nK, nT, 6, 6), dtype=torch.float64, device=dev)
    n_info = torch.empty((P, nK, nT), dtype=i32, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().usip_ransac_info_f64(
            _p(xyz), _p(count), S, L, _p(pairs), _p(frames), P, nK, _p(matches), _p(n_matches), cap, t_h, nT,
            float(threshold), int(seed) & (2 ** 64 - 1), _p(uniforms), _p(best_trial), _p(status), _p(info),
            _p(n_info), _stream()), "usip_ransac_info_f64")
    return info, n_info


def desc_match_mutual(desc, count, pairs, ks):
    """Mutual nearest-neighbour matches (FGR's AdvancedMatching cross-check) for every pair and K at once
    (include/usip_b200.h usip_desc_match_mutual_f64).  desc (S,L,D) f32, count (S,) i32, pairs (P,2) i32, all CUDA; ks
    ascending ints (host) -> (matches (P,nK,L,2) i32, n_matches (P,nK) i32), ascending by anchor row."""
    _req(desc, f32, "desc"); _req(count, i32, "count"); _req(pairs, i32, "pairs")
    S, L, D = desc.shape
    P = pairs.shape[0]
    if tuple(count.shape) != (S,) or pairs.dim() != 2 or pairs.shape[1] != 2:
        raise ValueError("count must be (%d,) and pairs (P, 2)" % S)
    ks_h = (ctypes.c_int32 * len(ks))(*[int(v) for v in ks])
    matches = torch.empty((P, len(ks), L, 2), dtype=i32, device=desc.device)
    n = torch.empty((P, len(ks)), dtype=i32, device=desc.device)
    with torch.cuda.device(desc.device):
        check(_lib.load().usip_desc_match_mutual_f64(_p(desc), _p(count), S, L, D, _p(pairs), P, ks_h, len(ks),
                                                     _p(matches), _p(n), _stream()), "usip_desc_match_mutual_f64")
    return matches, n


def fgr(xyz, count, pairs, ks, matches, n_matches, threshold=0.2, seed=0):
    """Fast Global Registration of every pair and K at once (include/usip_b200.h usip_fgr_f64).  xyz (S,L,3) f32, count
    (S,) i32, pairs (P,2) i32, matches / n_matches from desc_match_mutual, all CUDA; ks the same ascending ints (host):
    fragment f of a (pair, K) is its scan's first min(K, count, L) rows -> dict of Rt (P,nK,3,4) f64, n_tuples,
    n_inliers, status (P,nK) i32 and info (P,nK,6,6) f64."""
    _req(xyz, f32, "xyz"); _req(count, i32, "count"); _req(pairs, i32, "pairs")
    _req(matches, i32, "matches"); _req(n_matches, i32, "n_matches")
    S, L, _ = xyz.shape
    P, nK, cap = matches.shape[0], matches.shape[1], matches.shape[2]
    if tuple(xyz.shape) != (S, L, 3) or tuple(count.shape) != (S,) or tuple(pairs.shape) != (P, 2):
        raise ValueError("xyz must be (S, L, 3), count (S,) and pairs (P, 2)")
    if tuple(matches.shape) != (P, nK, cap, 2) or tuple(n_matches.shape) != (P, nK) or len(ks) != nK:
        raise ValueError("matches must be (P, nK, cap, 2) and n_matches (P, nK), nK = len(ks)")
    ks_h = (ctypes.c_int32 * nK)(*[int(v) for v in ks])
    dev = xyz.device
    e = lambda: torch.empty((P, nK), dtype=i32, device=dev)
    out = {"Rt": torch.empty((P, nK, 3, 4), dtype=torch.float64, device=dev), "n_tuples": e(), "n_inliers": e(),
           "info": torch.empty((P, nK, 6, 6), dtype=torch.float64, device=dev), "status": e()}
    with torch.cuda.device(dev):
        check(_lib.load().usip_fgr_f64(
            _p(xyz), _p(count), S, L, _p(pairs), P, ks_h, nK, _p(matches), _p(n_matches), cap,
            int(seed) & (2 ** 64 - 1), float(threshold), _p(out["Rt"]), _p(out["n_tuples"]), _p(out["n_inliers"]),
            _p(out["info"]), _p(out["status"]), _stream()), "usip_fgr_f64")
    return out


def fragment_overlap(xyz, offsets, jobs, Rt, radius=0.2):
    """register2Fragments.m's aligned-point count (include/usip_b200.h usip_fragment_overlap_f32): xyz (R,3) f32 CUDA,
    every fragment's rows packed; offsets (n_frags + 1,) ints and jobs (J, 2) ints (fragment a, fragment b), host
    (numpy or lists); Rt (J,3,4) f64 CUDA mapping b into a's frame -> hits (J,) i32 CUDA, the number of points of a
    within `radius` of some mapped point of b."""
    _req(xyz, f32, "xyz"); _req(Rt, torch.float64, "Rt")
    offsets = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
    jobs = np.ascontiguousarray(jobs, dtype=np.int32).reshape(-1, 2)
    nf, J = len(offsets) - 1, len(jobs)
    if xyz.dim() != 2 or xyz.shape[1] != 3 or nf < 1 or int(offsets[-1]) != xyz.shape[0]:
        raise ValueError("xyz must be (offsets[-1], 3) with at least one fragment")
    if tuple(Rt.shape) != (J, 3, 4):
        raise ValueError("Rt must be (J, 3, 4)")
    hits = torch.empty((J,), dtype=i32, device=xyz.device)
    if J == 0:
        return hits
    lib = _lib.load()
    nbytes = int(lib.usip_fragment_overlap_scratch_bytes(int(offsets[-1]), nf, J))
    scratch = torch.empty(((nbytes + 15) // 16, 4), dtype=i32, device=xyz.device)
    with torch.cuda.device(xyz.device):
        check(lib.usip_fragment_overlap_f32(_p(xyz), offsets.ctypes.data, nf, jobs.ctypes.data, _p(Rt), J,
                                            float(radius), _p(scratch), nbytes, _p(hits), _stream()),
              "usip_fragment_overlap_f32")
    return hits


def ransac_uniforms(T, seed=0, device="cuda"):
    """The uniforms ransac_rt draws for trials 0..T-1 from `seed` -> (T, 3) f64 CUDA."""
    out = torch.empty((int(T), 3), dtype=torch.float64, device=device)
    with torch.cuda.device(out.device):
        check(_lib.load().usip_ransac_uniforms(int(seed) & (2 ** 64 - 1), int(T), _p(out), _stream()),
              "usip_ransac_uniforms")
    return out


def nms(keypoints, sigmas, radius):
    """keypoints (B,3,M) f32, sigmas (B,M) f32 -> (idx (B,M) i32 kept indices in emission order, -1 padded; count (B,) i32)."""
    _req(keypoints, f32, "keypoints"); _req(sigmas, f32, "sigmas")
    B, _, M = keypoints.shape
    idx = torch.empty((B, M), dtype=i32, device=keypoints.device)
    cnt = torch.empty((B,), dtype=i32, device=keypoints.device)
    with torch.cuda.device(keypoints.device):
        check(_lib.load().usip_nms_f32(_p(keypoints), _p(sigmas), float(radius), _p(idx), _p(cnt), B, M, _stream()), "usip_nms_f32")
    return idx, cnt


class HcGrid:
    """The cell grid of a batch of test clouds (usip_hc_grid_build): pc (B,3,N) f32 CUDA and its scratch.  The radius
    passes below take it so that one build serves every pass of a batch."""

    def __init__(self, pc, scratch, nbytes):
        self.pc, self.scratch, self.nbytes = pc, scratch, nbytes
        self.B, self.N = pc.shape[0], pc.shape[2]


def hc_grid(pc):
    """usip_hc_grid_build: pc (B,3,N) f32 CUDA -> HcGrid."""
    _req(pc, f32, "pc")
    if pc.dim() != 3 or pc.shape[1] != 3:
        raise ValueError("pc must be (B, 3, N)")
    B, _, N = pc.shape
    lib = _lib.load()
    nbytes = int(lib.usip_hc_grid_scratch_bytes(B, N))
    if nbytes == 0:
        raise ValueError("hc_grid: B=%d, N=%d is outside the library's limits (include/usip_b200.h)" % (B, N))
    scratch = torch.empty(((nbytes + 15) // 16, 4), dtype=i32, device=pc.device)
    with torch.cuda.device(pc.device):
        check(lib.usip_hc_grid_build(_p(pc), _p(scratch), nbytes, B, N, _stream()), "usip_hc_grid_build")
    return HcGrid(pc, scratch, nbytes)


def iss_saliency(grid, salient_radius, gamma_21, gamma_32, min_neighbors, want_eig=False):
    """usip_iss_saliency_f64 -> (saliency (B,N) f64, count (B,N) i32 = |N_rs|, eig (B,N,3) f64 descending or None)."""
    pc, B, N = grid.pc, grid.B, grid.N
    sal = torch.empty((B, N), dtype=torch.float64, device=pc.device)
    cnt = torch.empty((B, N), dtype=i32, device=pc.device)
    eig = torch.empty((B, N, 3), dtype=torch.float64, device=pc.device) if want_eig else None
    with torch.cuda.device(pc.device):
        check(_lib.load().usip_iss_saliency_f64(_p(pc), _p(grid.scratch), grid.nbytes, B, N, float(salient_radius),
                                                float(gamma_21), float(gamma_32), int(min_neighbors), _p(sal),
                                                _p(cnt), _p(eig), _stream()), "usip_iss_saliency_f64")
    return sal, cnt, eig


def harris3d_response(grid, radius):
    """usip_harris3d_response_f64 -> (response (B,N) f64, count (B,N) i32 = |N_r|, normals (B,N,3) f64)."""
    pc, B, N = grid.pc, grid.B, grid.N
    resp = torch.empty((B, N), dtype=torch.float64, device=pc.device)
    cnt = torch.empty((B, N), dtype=i32, device=pc.device)
    nrm = torch.empty((B, N, 3), dtype=torch.float64, device=pc.device)
    with torch.cuda.device(pc.device):
        check(_lib.load().usip_harris3d_response_f64(_p(pc), _p(grid.scratch), grid.nbytes, B, N, float(radius),
                                                     _p(nrm), _p(resp), _p(cnt), _stream()),
              "usip_harris3d_response_f64")
    return resp, cnt, nrm


def hc_nonmax(grid, score, radius, threshold, strict, min_neighbors):
    """usip_hc_nonmax: score (B,N) f64 CUDA -> (flag (B,N) i32, count (B,N) i32 = |N_r|)."""
    _req(score, torch.float64, "score")
    pc, B, N = grid.pc, grid.B, grid.N
    if tuple(score.shape) != (B, N):
        raise ValueError("score must be (B, N)")
    flag = torch.empty((B, N), dtype=i32, device=pc.device)
    cnt = torch.empty((B, N), dtype=i32, device=pc.device)
    with torch.cuda.device(pc.device):
        check(_lib.load().usip_hc_nonmax(_p(pc), _p(grid.scratch), grid.nbytes, B, N, _p(score), float(radius),
                                         float(threshold), 1 if strict else 0, int(min_neighbors), _p(flag), _p(cnt),
                                         _stream()), "usip_hc_nonmax")
    return flag, cnt


def hc_select(flag, B, N, L, seed=0, step=0, device="cuda"):
    """usip_hc_select: flag (B,N) i32 CUDA or None (random) -> (order (B,L) i32, count (B,) i32 flagged rows)."""
    if flag is not None:
        _req(flag, i32, "flag")
        if tuple(flag.shape) != (B, N):
            raise ValueError("flag must be (B, N)")
        device = flag.device
    order = torch.empty((B, int(L)), dtype=i32, device=device)
    cnt = torch.empty((B,), dtype=i32, device=device)
    with torch.cuda.device(order.device):
        check(_lib.load().usip_hc_select(_p(flag), B, N, int(L), int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1),
                                         _p(order), _p(cnt), _stream()), "usip_hc_select")
    return order, cnt


def knn_gather(src, idx):
    _req(src, f32, "som_node"); _req(idx, i32, "som_node_knn_I")
    B, C, N = src.shape
    M, K = idx.shape[1], idx.shape[2]
    out = torch.empty((B, C, M, K), dtype=f32, device=src.device)
    check(_lib.load().usip_knn_gather_f32(_p(src), _p(idx), _p(out), B, C, N, M, K, _stream()), "usip_knn_gather_f32")
    return out


# ----------------------------------------------------------------------------- grouping
def som_assign(xyz, node, count=None, method="auto"):
    """Nearest node of every point (som.query_topk, k = 1).  method: "auto" | "brute" | "grid" (identical results): the grid
    path bins the nodes into cells and searches the shells around each point (usip_som_assign_grid_f32)."""
    _req(xyz, f32, "x"); _req(node, f32, "node")
    B, _, N = xyz.shape
    M = node.shape[2]
    min_idx = torch.empty((B, N), dtype=i32, device=xyz.device)
    if count is None:
        count = torch.zeros((B, M), dtype=i32, device=xyz.device)
    lib = _lib.load()
    if method == "grid" or (method == "auto" and 64 <= M <= 1024 and N >= 1024):
        nbytes = int(lib.usip_som_assign_grid_scratch_bytes(B, M))
        scratch = torch.empty(((nbytes + 15) // 16, 4), dtype=i32, device=xyz.device)
        check(lib.usip_som_assign_grid_f32(_p(xyz), _p(node), _p(min_idx), _p(count), _p(scratch), nbytes, B, N, M, _stream()),
              "usip_som_assign_grid_f32")
        return min_idx, count
    check(lib.usip_som_assign_f32(_p(xyz), _p(node), _p(min_idx), _p(count), B, N, M, _stream()),
          "usip_som_assign_f32")
    return min_idx, count


def cluster_sort(min_idx, M):
    B, N = min_idx.shape
    dev = min_idx.device
    seg_off = torch.empty((B, M + 1), dtype=i32, device=dev)
    perm = torch.empty((B, N), dtype=i32, device=dev)
    row_seg = torch.empty((B, N), dtype=i32, device=dev)
    chunks = (N + 255) // 256
    scratch = torch.empty((B * chunks * M,), dtype=i32, device=dev)
    check(_lib.load().usip_cluster_sort(_p(min_idx), _p(seg_off), _p(perm), _p(row_seg), _p(scratch), B, N, M,
                                        _stream()), "usip_cluster_sort")
    return seg_off, perm, row_seg


def cluster_mean_decenter(xyz, feat, seg_off, perm, M, ldx=8):
    B, _, N = xyz.shape
    S = 0 if feat is None else feat.shape[1]
    cmean = torch.empty((B, 3, M), dtype=f32, device=xyz.device)
    x_aug = torch.empty((B * N, ldx), dtype=f32, device=xyz.device)
    check(_lib.load().usip_cluster_mean_decenter(_p(xyz), _p(feat) if S else None, _p(seg_off), _p(perm), _p(cmean),
                                                 _p(x_aug), ldx, B, S, N, M, _stream()), "usip_cluster_mean_decenter")
    return cmean, x_aug


def segmax(X, C, seg_off, perm, B, N, M, out=None, arg=None, want_arg=True):
    ldx = X.stride(0)
    if out is None:
        out = torch.empty((B * M, C), dtype=f32, device=X.device)
    if arg is None and want_arg:
        arg = torch.empty((B * M, C), dtype=i32, device=X.device)
    check(_lib.load().usip_segmax(_p(X), ldx, _p(seg_off), _p(perm), _p(out), out.stride(0), _p(arg), B, N, M, C,
                                  _stream()), "usip_segmax")
    return out, arg


def knn_nodes(pts, K):
    _req(pts, f32, "pts")
    B, _, M = pts.shape
    out = torch.empty((B, M, K), dtype=i32, device=pts.device)
    check(_lib.load().usip_knn_nodes(_p(pts), _p(out), B, M, K, _stream()), "usip_knn_nodes")
    return out


# ----------------------------------------------------------------------------- shared-MLP stack
def layer_fwd(X, W, bias, P, Cin, Cout, ldx=None, ldw=None, in_scale=None, in_shift=None, in_relu=False,
              addend=None, add_index=None, add_group=0, Y=None, ldy=None, stat_partial=None,
              gmax=None, gmin=None, garg_max=None, garg_min=None, group=0, precision=0, tc_ws=None, tc_packed=False, w_transposed=False, debug_flags=0, debug_clocks=None):
    """Launches one layer; returns the LayerDesc it launched with."""
    d = LayerDesc()
    d.X = X.data_ptr(); d.ldx = X.stride(0) if ldx is None else ldx
    d.P = P; d.Cin = Cin; d.Cout = Cout
    d.W = W.data_ptr(); d.ldw = (W.stride(0) if ldw is None else ldw)
    d.w_transposed = 1 if w_transposed else 0
    d.bias = None if bias is None else bias.data_ptr()
    d.in_scale = None if in_scale is None else in_scale.data_ptr()
    d.in_shift = None if in_shift is None else in_shift.data_ptr()
    d.in_relu = 1 if in_relu else 0
    d.addend = None if addend is None else addend.data_ptr()
    d.ld_add = 0 if addend is None else addend.stride(0)
    d.add_index = None if add_index is None else add_index.data_ptr()
    d.add_group = add_group
    d.Y = None if Y is None else Y.data_ptr()
    d.ldy = 0 if Y is None else (Y.stride(0) if ldy is None else ldy)
    d.stat_partial = None if stat_partial is None else stat_partial.data_ptr()
    d.gmax = None if gmax is None else gmax.data_ptr()
    d.gmin = None if gmin is None else gmin.data_ptr()
    d.garg_max = None if garg_max is None else garg_max.data_ptr()
    d.garg_min = None if garg_min is None else garg_min.data_ptr()
    d.group = group
    d.precision = precision
    d.debug_flags = debug_flags
    d.debug_clocks = debug_clocks.data_ptr() if debug_clocks is not None else None
    if precision == 1:
        if tc_ws is None:
            tc_ws = torch.empty((2 * Cin * Cout,), dtype=f32, device=X.device)
        d.tc_workspace = tc_ws.data_ptr(); d.tc_workspace_bytes = tc_ws.numel() * 4
        d.tc_weights_packed = 1 if tc_packed else 0
    check(_lib.load().usip_layer_fwd(ctypes.byref(d), _stream()),
          "usip_layer_fwd_tc" if (precision == 1 and not tc_packed) else "usip_layer_fwd")
    return d


def bn_finalize(stat_partial, ntiles, count, C, gamma, beta, eps, momentum, running_mean, running_var,
                scale, shift, save_mean=None, save_invstd=None):
    check(_lib.load().usip_bn_finalize(_p(stat_partial), ntiles, int(count), C, _p(gamma), _p(beta), float(eps),
                                       float(momentum), _p(running_mean), _p(running_var), _p(scale), _p(shift),
                                       _p(save_mean), _p(save_invstd), _stream()), "usip_bn_finalize")


def bn_eval_affine(gamma, beta, running_mean, running_var, eps, scale, shift):
    C = gamma.numel()
    check(_lib.load().usip_bn_eval_affine(_p(gamma), _p(beta), _p(running_mean), _p(running_var), float(eps), C,
                                          _p(scale), _p(shift), _stream()), "usip_bn_eval_affine")


def knn_combine(Z, pts, knn_idx, W, ldw, bias, Y, stat_partial, B, M, K, Cout):
    check(_lib.load().usip_knn_combine(_p(Z), Z.stride(0), _p(pts), _p(knn_idx), _p(W), ldw, _p(bias), _p(Y),
                                       Y.stride(0), _p(stat_partial), B, M, K, Cout, _stream()), "usip_knn_combine")


def group_select(gmax, gmin, scale, shift, out, Q, C):
    check(_lib.load().usip_group_select(_p(gmax), _p(gmin), _p(scale), _p(shift), _p(out), out.stride(0), Q, C,
                                        _stream()), "usip_group_select")


def group_max_combine(gmax, ratio, gmin=None):
    """[Q*ratio, C] per-sub-group max (and min) -> [Q, C]: the max (min) over each run of `ratio` consecutive rows."""
    _req(gmax, f32, "gmax")
    if gmin is not None:
        _req(gmin, f32, "gmin")
        if gmin.shape != gmax.shape:
            raise ValueError("gmin %s must have gmax's shape %s" % (tuple(gmin.shape), tuple(gmax.shape)))
    R, C = gmax.shape
    if ratio < 1 or R % ratio != 0:
        raise ValueError("group_max_combine: ratio %d must divide the %d rows" % (ratio, R))
    Q = R // ratio
    omax = torch.empty((Q, C), dtype=f32, device=gmax.device)
    omin = None if gmin is None else torch.empty((Q, C), dtype=f32, device=gmax.device)
    check(_lib.load().usip_group_max_combine(_p(gmax), _p(gmin), _p(omax), _p(omin), int(ratio), Q, C, _stream()),
          "usip_group_max_combine")
    return omax, omin


def group_max_combine_arg(gmax, ratio, gmin=None, amax=None, amin=None, sub=1):
    """group_max_combine with arg outputs -> (omax, omin, oamax, oamin), oamax / oamin [Q, C] i32 the row of the result in
    the whole group of ratio * sub rows: r * sub + amax[q*ratio + r] with the sub-groups' row-in-sub-group args amax /
    amin, r without them (r: the first of the `ratio` input rows holding the max / min, 0 when none beats -inf / +inf)."""
    _req(gmax, f32, "gmax")
    for name, t, dt in (("gmin", gmin, f32), ("amax", amax, i32), ("amin", amin, i32)):
        if t is not None:
            _req(t, dt, name)
            if t.shape != gmax.shape:
                raise ValueError("%s %s must have gmax's shape %s" % (name, tuple(t.shape), tuple(gmax.shape)))
    if amin is not None and (amax is None or gmin is None):
        raise ValueError("group_max_combine_arg: amin needs amax and gmin")
    if amax is not None and gmin is not None and amin is None:
        raise ValueError("group_max_combine_arg: the sub-group args of gmin (amin) are missing")
    R, C = gmax.shape
    if ratio < 1 or R % ratio != 0:
        raise ValueError("group_max_combine_arg: ratio %d must divide the %d rows" % (ratio, R))
    Q = R // ratio
    dev = gmax.device
    omax = torch.empty((Q, C), dtype=f32, device=dev)
    oamax = torch.empty((Q, C), dtype=i32, device=dev)
    omin = None if gmin is None else torch.empty((Q, C), dtype=f32, device=dev)
    oamin = None if gmin is None else torch.empty((Q, C), dtype=i32, device=dev)
    check(_lib.load().usip_group_max_combine_arg(_p(gmax), _p(gmin), _p(amax), _p(amin), _p(omax), _p(omin), _p(oamax),
                                                 _p(oamin), int(ratio), int(sub), Q, C, _stream()),
          "usip_group_max_combine_arg")
    return omax, omin, oamax, oamin


def head_finalize(out4, cluster_mean, lb, B, M):
    kp = torch.empty((B, 3, M), dtype=f32, device=out4.device)
    sig = torch.empty((B, M), dtype=f32, device=out4.device)
    check(_lib.load().usip_head_finalize(_p(out4), out4.stride(0), _p(cluster_mean), float(lb), _p(kp), _p(sig), B, M,
                                         _stream()), "usip_head_finalize")
    return kp, sig


# ----------------------------------------------------------------------------- losses
# databases at least this large go through the cell grid (usip_pairwise_min_grid_f32); smaller ones stay brute force
PAIRWISE_MIN_GRID_FROM = 4096


def pairwise_min(a, b, method="auto"):
    """a (B,3,Ma), b (B,3,Nb) -> (min_d (B,Ma) f32, arg (B,Ma) i32).  method: "auto" | "brute" | "grid" (same result)."""
    _req(a, f32, "a"); _req(b, f32, "b")
    B, _, Ma = a.shape
    Nb = b.shape[2]
    d = torch.empty((B, Ma), dtype=f32, device=a.device)
    arg = torch.empty((B, Ma), dtype=i32, device=a.device)
    lib = _lib.load()
    if method == "grid" or (method == "auto" and Nb >= PAIRWISE_MIN_GRID_FROM):
        nbytes = int(lib.usip_pairwise_min_grid_scratch_bytes(B, Nb))
        scratch = torch.empty(((nbytes + 15) // 16, 4), dtype=i32, device=a.device)
        check(lib.usip_pairwise_min_grid_f32(_p(a), _p(b), _p(d), _p(arg), _p(scratch), nbytes, B, Ma, Nb, _stream()),
              "usip_pairwise_min_grid_f32")
        return d, arg
    packed = torch.empty((B, Ma), dtype=torch.int64, device=a.device)
    check(lib.usip_pairwise_min_f32(_p(a), _p(b), _p(d), _p(arg), _p(packed), B, Ma, Nb, _stream()),
          "usip_pairwise_min_f32")
    if Nb <= 2048:
        _lib.LAUNCHES[0] -= 2          # small databases take the single-kernel path (no init / finish launches)
    return d, arg


def chamfer_prob_reduce(d_sd, i_sd, d_ds, i_ds, sig_src, sig_dst):
    B, M = d_sd.shape
    N = d_ds.shape[1]
    out = torch.empty((3,), dtype=f32, device=d_sd.device)
    check(_lib.load().usip_chamfer_prob_reduce(_p(d_sd), _p(i_sd), _p(d_ds), _p(i_ds), _p(sig_src), _p(sig_dst),
                                               _p(out), B, M, N, _stream()), "usip_chamfer_prob_reduce")
    return out


def transform_points(kp, R, scale, shift):
    B, _, M = kp.shape
    out = torch.empty_like(kp)
    check(_lib.load().usip_transform_points(_p(kp), _p(R), _p(scale), _p(shift), _p(out), B, M, _stream()),
          "usip_transform_points")
    return out


def mean_scale(d, alpha):
    out = torch.empty((1,), dtype=f32, device=d.device)
    check(_lib.load().usip_mean_scale(_p(d), d.numel(), float(alpha), _p(out), _stream()), "usip_mean_scale")
    return out


# DescCGFLoss kernels (include/usip_b200.h): the positive keypoints of a cloud are staged in shared memory, and the backward
# keeps D/32 descriptor channels per lane in registers
CGF_MAX_M = 2048
CGF_MAX_D = 512


def desc_cgf_check(anc_kp, pos_kp, anc_desc, pos_desc, sigma, draws):
    """Host-side argument check of desc_cgf (no device needed): float32, contiguous, shapes (B,3,M), (B,D,M), (B,M) and
    the draws (B,M,M), (B,M,M), (B,M); M <= CGF_MAX_M, D a multiple of 4 in [4, CGF_MAX_D].  -> (B, M, D)"""
    B, _, M = anc_kp.shape
    D = anc_desc.shape[1]
    want = dict(anc_kp=(B, 3, M), pos_kp=(B, 3, M), anc_desc=(B, D, M), pos_desc=(B, D, M), sigma=(B, M),
                u_near=(B, M, M), u_out=(B, M, M), u_sel=(B, M))
    got = dict(anc_kp=anc_kp, pos_kp=pos_kp, anc_desc=anc_desc, pos_desc=pos_desc, sigma=sigma, u_near=draws[0],
               u_out=draws[1], u_sel=draws[2])
    for name, t in got.items():
        if t.dtype != f32:
            raise ValueError("desc_cgf: %s must be float32, got %s" % (name, t.dtype))
        if not t.is_contiguous():
            raise ValueError("desc_cgf: %s must be contiguous" % name)
        if tuple(t.shape) != want[name]:
            raise ValueError("desc_cgf: %s has shape %s, expected %s" % (name, tuple(t.shape), want[name]))
    if B < 1 or M < 1:
        raise ValueError("desc_cgf: empty batch (B=%d, M=%d)" % (B, M))
    if M > CGF_MAX_M:
        raise ValueError("desc_cgf: M=%d keypoints exceed the %d the kernel stages in shared memory" % (M, CGF_MAX_M))
    if D % 4 != 0 or not 4 <= D <= CGF_MAX_D:
        raise ValueError("desc_cgf: descriptor length D=%d must be a multiple of 4 in [4, %d]" % (D, CGF_MAX_D))
    return B, M, D


def desc_cgf(anc_kp, pos_kp, anc_desc, pos_desc, sigma, draws, radius, gamma, sigma_max):
    """DescCGFLoss forward (usip_desc_cgf_f32) -> loss (B,M), active (B), saved = (sel (B,M,4) i32, aux (B,M,4) f32,
    cloud (B,2) f32) for desc_cgf_bwd."""
    B, M, D = desc_cgf_check(anc_kp, pos_kp, anc_desc, pos_desc, sigma, draws)
    for name, t in (("anc_kp", anc_kp), ("anc_desc", anc_desc), ("u_near", draws[0])):
        _req(t, f32, name)
    dev = anc_kp.device
    loss = torch.empty((B, M), dtype=f32, device=dev)
    active = torch.empty((B,), dtype=f32, device=dev)
    sel = torch.empty((B, M, 4), dtype=i32, device=dev)
    aux = torch.empty((B, M, 4), dtype=f32, device=dev)
    cloud = torch.empty((B, 2), dtype=f32, device=dev)
    check(_lib.load().usip_desc_cgf_f32(_p(anc_kp), _p(pos_kp), _p(anc_desc), _p(pos_desc), _p(sigma), _p(draws[0]),
                                        _p(draws[1]), _p(draws[2]), float(radius), float(gamma), float(sigma_max), _p(loss),
                                        _p(active), _p(sel), _p(aux), _p(cloud), B, M, D, _stream()), "usip_desc_cgf_f32")
    return loss, active, (sel, aux, cloud)


def desc_cgf_bwd(anc_desc, pos_desc, sigma, saved, g_loss, sigma_max):
    """DescCGFLoss backward (usip_desc_cgf_bwd) -> g_anc, g_pos (B,D,M)."""
    sel, aux, cloud = saved
    B, D, M = anc_desc.shape
    g = g_loss.contiguous().float()
    if tuple(g.shape) != (B, M):
        raise ValueError("desc_cgf_bwd: g_loss has shape %s, expected %s" % (tuple(g.shape), (B, M)))
    g_anc = torch.empty_like(anc_desc)
    g_pos = torch.empty_like(pos_desc)
    check(_lib.load().usip_desc_cgf_bwd(_p(anc_desc), _p(pos_desc), _p(sigma), _p(sel), _p(aux), _p(cloud), _p(g),
                                        float(sigma_max), _p(g_anc), _p(g_pos), B, M, D, _stream()), "usip_desc_cgf_bwd")
    return g_anc, g_pos
