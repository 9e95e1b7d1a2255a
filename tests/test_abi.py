"""CPU-side checks of the drop-in boundary: libusip_b200.so loads without a GPU, exports every symbol that
include/usip_b200.h declares, and the ctypes binding covers exactly that set (no compute calls here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "usip_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(usip_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    from usip_b200 import _lib
    lib = _lib.load()
    declared = _declared()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), "declared in usip_b200.h but not exported: " + name
    assert sorted(_lib.SIGNATURES) == declared, (set(declared) ^ set(_lib.SIGNATURES))
    assert lib.usip_abi_version() == 1
    assert lib.usip_layer_tile_rows() == 128


def test_layer_desc_layout_matches_c_struct():
    """sizeof/offsets of the ctypes mirror must match the C struct (compiled with gcc here)."""
    import subprocess, tempfile
    from usip_b200._lib import LayerDesc
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "usip_b200.h"
int main(){ printf("%zu %zu %zu %zu %zu %zu\n", sizeof(usip_layer_desc), offsetof(usip_layer_desc, W),
  offsetof(usip_layer_desc, addend), offsetof(usip_layer_desc, Y), offsetof(usip_layer_desc, gmax),
  offsetof(usip_layer_desc, precision)); return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = [int(v) for v in subprocess.check_output([exe]).split()]
    assert out == [ctypes.sizeof(LayerDesc), LayerDesc.W.offset, LayerDesc.addend.offset, LayerDesc.Y.offset,
                   LayerDesc.gmax.offset, LayerDesc.precision.offset]


def _misaligned_calls():
    """One call per (entry point, float4 operand) of the backward kernels, segmax and knn_combine with that operand 4
    bytes off a 16-byte boundary; every other pointer is aligned.  The addresses are never dereferenced: the argument
    check runs first."""
    from usip_b200 import _lib
    lib = _lib.load()
    A = 0x100000

    def ptrs(n, bad):
        return [ctypes.c_void_p(A + 0x10000 * i + (4 if i == bad else 0)) for i in range(n)]

    calls = []
    for bad in range(7):      # G, Y, scale, shift, mean, invstd, part
        G, Y, sc, sh, mu, iv, part = ptrs(7, bad)
        calls.append(("bn_bwd_reduce", bad, lambda G=G, Y=Y, sc=sc, sh=sh, mu=mu, iv=iv, part=part:
                      lib.usip_bn_bwd_reduce(G, 64, Y, 64, sc, sh, mu, iv, 1, part, 1000, 64, None)))
        calls.append(("bn_bwd_reduce/C=48", bad, lambda G=G, Y=Y, sc=sc, sh=sh, mu=mu, iv=iv, part=part:
                      lib.usip_bn_bwd_reduce(G, 48, Y, 48, sc, sh, mu, iv, 1, part, 1000, 48, None)))
    for bad in range(9):      # G, Y, scale, shift, mean, invstd, c1, c2, GY
        G, Y, sc, sh, mu, iv, c1, c2, GY = ptrs(9, bad)
        for C in (64, 96):
            calls.append(("bn_bwd_apply/C=%d" % C, bad, lambda G=G, Y=Y, sc=sc, sh=sh, mu=mu, iv=iv, c1=c1, c2=c2, GY=GY, C=C:
                          lib.usip_bn_bwd_apply(G, C, Y, C, sc, sh, mu, iv, c1, c2, 1, GY, C, 1000, C, None)))
    for bad in range(9):      # Y, gz, argsel, scale, mean, invstd, c1, c2, GY
        Y, gz, a, sc, mu, iv, c1, c2, GY = ptrs(9, bad)
        calls.append(("groupmax_bwd_apply", bad, lambda Y=Y, gz=gz, a=a, sc=sc, mu=mu, iv=iv, c1=c1, c2=c2, GY=GY:
                      lib.usip_groupmax_bwd_apply(Y, 64, gz, a, sc, mu, iv, c1, c2, GY, 64, 16, 1600, 64, None)))
    for bad in range(2):      # G, out
        G, out = ptrs(2, bad)
        calls.append(("group_sum", bad, lambda G=G, out=out: lib.usip_group_sum(G, 64, out, 64, 16, 100, 64, None)))
        seg = ctypes.c_void_p(A + 0x80000)
        calls.append(("seg_sum", bad, lambda G=G, out=out, seg=seg: lib.usip_seg_sum(G, 64, seg, out, 64, 2, 500, 8, 64, None)))
    G, = ptrs(1, 0)
    calls.append(("head_bwd", 0, lambda G=G: lib.usip_head_bwd(None, None, ctypes.c_void_p(A + 0x40000), 4, G, 2, 10, None)))
    GY, = ptrs(1, 0)
    aligned = ctypes.c_void_p(A + 0x40000)
    calls.append(("knn_combine_bwd", 0, lambda GY=GY: lib.usip_knn_combine_bwd(GY, 128, aligned, aligned, aligned, 128, aligned,
                                                                                128, 1, 32, 16, 128, None)))
    # forward kernels with float4 / int4 operands
    for bad in range(3):      # X, pooled, arg
        X, pooled, arg = ptrs(3, bad)
        calls.append(("segmax", bad, lambda X=X, pooled=pooled, arg=arg:
                      lib.usip_segmax(X, 64, aligned, aligned, pooled, 64, arg, 2, 500, 8, 64, None)))
    for bad in range(2):      # Z, Y
        Z, Y = ptrs(2, bad)
        calls.append(("knn_combine", bad, lambda Z=Z, Y=Y:
                      lib.usip_knn_combine(Z, 128, aligned, aligned, aligned, 128, aligned, Y, 128, aligned, 1, 32, 16, 128, None)))
    return lib, calls


def test_backward_entry_points_reject_misaligned_operands():
    """A misaligned float4 operand is refused on the host (-1, no launch) -- it used to reach a kernel and fault the device."""
    lib, calls = _misaligned_calls()
    for name, bad, fn in calls:
        assert fn() == -1, (name, bad)
        assert b"aligned" in lib.usip_last_error(), (name, bad, lib.usip_last_error())


def test_neighbour_entry_points_refuse_before_launch():
    """Sizes the neighbour-search, sampling and NMS kernels cannot take are refused on the host (-1, no launch): the
    addresses are never dereferenced, and a launch on a machine without a GPU would fail with a CUDA error instead."""
    from usip_b200 import _lib
    lib = _lib.load()
    a = [ctypes.c_void_p(0x100000 + 0x10000 * i) for i in range(8)]
    calls = [
        ("nms M = 8534", lambda: lib.usip_nms_f32(a[0], a[1], 1.0, a[2], a[3], 1, 8534, None), b"M too large"),
        ("fps Ns = 8193", lambda: lib.usip_fps_f32(a[0], a[1], a[2], a[3], 1, 8193, 16, None), b"8192"),
        ("knn_group K > N", lambda: lib.usip_knn_group_f32(a[0], a[1], a[2], a[3], a[4], a[5], 8, 1, 4, 100, 16, 101, None),
         b"K <= N"),
        ("knn_group S = 6", lambda: lib.usip_knn_group_f32(a[0], a[1], a[2], a[3], a[4], a[5], 16, 1, 6, 100, 16, 8, None),
         b"S <= 5"),
        ("cluster_sort M too large", lambda: lib.usip_cluster_sort(a[0], a[1], a[2], a[3], a[4], 1, 1000, 50177, None),
         b"M too large"),
    ]
    for name, fn, msg in calls:
        assert fn() == -1, name
        assert msg in lib.usip_last_error(), (name, lib.usip_last_error())


def test_product_path_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from usip_b200 import index_max
    with pytest.raises(RuntimeError):
        index_max.forward_cuda_shared_mem(torch.zeros(1, 1, 4), torch.zeros(1, 4, dtype=torch.int32), 2)


def test_product_code_never_imports_oracle():
    """oracle/ is test infrastructure: nothing under usip_b200/ may import or execute it."""
    pkg = os.path.join(ROOT, "usip_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), os.path.join(dp, f)
                assert "usip_oracle" not in txt or f == "index_max.py", os.path.join(dp, f)
