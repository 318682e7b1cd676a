"""CPU tests of the drop-in boundary: the C-ABI library loads without a GPU, exports every symbol
include/frcnn_b200.h declares, and the host-side mirror (models/, compat shim) imports with the
reference's names and signatures.  No compute call is made here."""
import ctypes
import inspect
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "frcnn_b200.h")


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "chainer-faster-rcnn_b200", "csrc"), "-j4"])
    return _lib.load()


def _declared_symbols():
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(_nms|frcnn_[a-z0-9_]+)\s*\(", txt)))


def test_library_loads_and_exports_every_declared_symbol(lib):
    from frcnn_b200 import _lib
    syms = _declared_symbols()
    assert len(syms) >= 18
    for s in syms:
        assert hasattr(lib, s), "missing export: " + s
    assert set(_lib.SIGNATURES) == set(syms), set(_lib.SIGNATURES) ^ set(syms)
    assert lib.frcnn_version() >= 100
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for s in syms:
        assert re.search(r"\sT\s+%s$" % re.escape(s), out, flags=re.M), s


def test_every_conv_gemm_instantiation_has_a_dispatch_matrix_case():
    """The FRCNN_DISPATCH(...) lines of conv_gemm_sm90.cu are exactly the parameter list of the GPU dispatch-matrix test
    (tests/test_conv_gemm_coverage_gpu.py), in the same order: an instantiation cannot be added without a test."""
    import test_conv_gemm_coverage_gpu as cov
    table = cov.parse_dispatch_table()
    assert len(table) == 25 and len(set(table)) == len(table)
    assert table == cov.DISPATCH
    assert set(cov.MATRIX_SHAPE) == set(cov.DISPATCH)


def test_conv_last_plan_reports_every_field(lib):
    from frcnn_b200 import ops
    assert lib.frcnn_conv2d_last_plan(None, 0) == len(ops.CONV_PLAN_FIELDS) == 12
    assert list(ops.conv_last_plan()) == list(ops.CONV_PLAN_FIELDS)


def test_no_hard_dependency_on_libcuda(lib):
    from frcnn_b200 import _lib
    out = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libcudart" not in out   # static cudart, driver API via the runtime


def test_argument_errors_are_reported_not_printed(lib):
    from frcnn_b200 import _lib
    # n > 16384 is rejected before any CUDA call: status + message, no crash
    r = lib.frcnn_nms(None, 20000, 0.7, 0, 0, None, ctypes.c_void_p(1), None, 0, None)
    assert r == _lib.ERR_ARG and "16384" in _lib.last_error()
    assert lib.frcnn_nms_workspace_bytes(6000) > 6000 * 94 * 8
    assert lib.frcnn_proposals_workspace_bytes(9, 38, 63, 6000) > 4_000_000


def test_dropin_modules_mirror_the_reference_api():
    from frcnn_b200 import dropin
    dropin.install()
    import chainer
    from models import bbox_transform, cpu_nms, faster_rcnn, generate_anchors, gpu_nms, proposal_layer
    from models import region_proposal_network, vgg16
    PL = proposal_layer.ProposalLayer
    assert (PL.RPN_NMS_THRESH, PL.TRAIN_RPN_PRE_NMS_TOP_N, PL.TRAIN_RPN_POST_NMS_TOP_N,
            PL.TEST_RPN_PRE_NMS_TOP_N, PL.TEST_RPN_POST_NMS_TOP_N, PL.RPN_MIN_SIZE) == (0.7, 12000, 2000, 6000, 300, 16)
    pl = PL()
    assert pl._num_anchors == 9 and pl.train is True and pl._pre_nms_top_n == 12000
    pl.train = False
    assert (pl._pre_nms_top_n, pl._post_nms_top_n) == (6000, 300)
    assert list(inspect.signature(PL.__call__).parameters) == ["self", "rpn_cls_prob", "rpn_bbox_pred", "img_info"]
    assert list(inspect.signature(region_proposal_network.RegionProposalNetwork.__call__).parameters) == \
        ["self", "x", "img_info", "gt_boxes"]
    sig = inspect.signature(faster_rcnn.FasterRCNN.__init__)
    assert list(sig.parameters)[1:] == ["trunk_class", "rpn_in_ch", "rpn_mid_ch", "feat_stride", "anchor_ratios",
                                        "anchor_scales", "num_classes", "loss_lambda", "rpn_delta", "rcnn_delta"]
    assert sig.parameters["trunk_class"].default is vgg16.VGG16
    assert list(inspect.signature(faster_rcnn.FasterRCNN.__call__).parameters) == ["self", "x", "img_info", "gt_boxes"]
    for fn in ("bbox_transform", "bbox_transform_inv", "clip_boxes", "filter_boxes", "keep_inside"):
        assert callable(getattr(bbox_transform, fn))
    assert callable(cpu_nms.cpu_nms) and callable(gpu_nms.gpu_nms)
    # anchors: executed-reference known answer (SURVEY.md Q9)
    a = generate_anchors.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    assert a.dtype == np.float64 and a[0].tolist() == [-84, -40, 99, 55] and a[8].tolist() == [-168, -344, 183, 359]
    g = np.load(os.path.join(ROOT, "tests", "golden", "anchors.npz"))
    assert np.array_equal(generate_anchors.generate_anchors(), g["anchors_default_call"])
    assert np.array_equal(pl._generate_all_bbox(3, 4)[:9], a) and pl._generate_all_bbox(3, 4).shape == (108, 4)
    assert pl._generate_all_bbox(3, 4)[9 * 5 + 2].tolist() == (a[2] + [16, 16, 16, 16]).tolist()
    # model structure: the reference's checkpoint paths (SURVEY.md 5)
    m = faster_rcnn.FasterRCNN(trunk_class=vgg16.VGG16Prev)
    names = dict(m.namedparams())
    for k, shape in {"/trunk/conv1_1/W": (64, 3, 3, 3), "/trunk/conv5_3/b": (512,), "/RPN/rpn_conv_3x3/W": (512, 512, 3, 3),
                     "/RPN/rpn_cls_score/W": (18, 512, 1, 1), "/RPN/rpn_bbox_pred/b": (36,), "/fc6/W": (4096, 25088),
                     "/fc7/W": (4096, 4096), "/cls_score/W": (21, 4096), "/bbox_pred/W": (84, 4096)}.items():
        assert names[k].data.shape == shape, k
    assert len(names) == 2 * (13 + 3 + 4)
    assert m.rpn_train is False and m.rcnn_train is False
    m.rpn_train = True
    assert m.RPN.proposal_layer._pre_nms_top_n == 12000 and m.trunk.train is True
    m.rpn_train = False
    assert m.xp is np
    # type contract (models/faster_rcnn.py:76-90): batch 1, integer img_info, Variables
    with pytest.raises(AssertionError):
        m(chainer.Variable(np.zeros((2, 3, 32, 32), np.float32)), chainer.Variable(np.array([[32, 32]], np.int32)))
    with pytest.raises(AssertionError):
        m(chainer.Variable(np.zeros((1, 3, 32, 32), np.float32)), chainer.Variable(np.array([[32., 32.]], np.float32)))


def test_checkpoint_roundtrip_in_reference_npz_format(tmp_path):
    from frcnn_b200 import dropin
    dropin.install()
    from chainer import serializers
    from models.region_proposal_network import RegionProposalNetwork
    a, b = RegionProposalNetwork(), RegionProposalNetwork()
    path = str(tmp_path / "rpn.npz")
    serializers.save_npz(path, a)
    assert sorted(np.load(path).files) == ["rpn_bbox_pred/W", "rpn_bbox_pred/b", "rpn_cls_score/W", "rpn_cls_score/b",
                                           "rpn_conv_3x3/W", "rpn_conv_3x3/b"]
    v0 = b._version
    serializers.load_npz(path, b)
    assert np.array_equal(a.rpn_conv_3x3.W.data, b.rpn_conv_3x3.W.data) and b._version > v0


def test_product_path_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under chainer-faster-rcnn_b200/ may reference it."""
    pkg = os.path.join(ROOT, "chainer-faster-rcnn_b200")
    bad = []
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(d, f), errors="replace").read()
                if re.search(r"frcnn_oracle|oracle_c|import\s+build_ref|from\s+oracle", txt):
                    bad.append(os.path.join(d, f))
    assert not bad, bad


def test_compute_calls_fail_loudly_without_a_gpu():
    """No CPU fallback anywhere: on a box without a usable GPU a compute entry point returns FRCNN_ERR_CUDA with the CUDA
    runtime's message (it never computes on the host, never crashes), and the Python wrappers refuse host tensors."""
    import ctypes
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from frcnn_b200 import _lib, ops
    lib = _lib.load()
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)                         # noqa: E731
    b, q, o = np.zeros((4, 4)), np.zeros((2, 4)), np.zeros((4, 2))
    assert lib.frcnn_bbox_overlaps(p(b), 4, p(q), 2, p(o), None) == _lib.ERR_CUDA
    assert "CUDA" in _lib.last_error() or "cuda" in _lib.last_error()
    d, k = np.zeros((3, 5), np.float32), np.zeros(3, np.int32)
    assert lib.frcnn_cpu_nms_host(p(d), 3, 0.7, p(k), 0) < 0
    with pytest.raises(_lib.FrcnnError):
        ops.nms(torch.zeros((4, 5)), 0.7)
    with pytest.raises(_lib.FrcnnError):
        ops.cpu_nms_host(d, 0.7)


def test_header_is_plain_c_and_links_against_the_library(tmp_path):
    """include/frcnn_b200.h must be consumable from C (the reference-side bindings are Cython / cgo-style C callers):
    a C99 translation unit that takes the address of every declared entry point compiles with -Wall -Werror and links
    against libfrcnn_b200.so; running it prints the library version (no GPU needed)."""
    from frcnn_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = sorted(_lib.SIGNATURES)
    src = ['#include <stdio.h>', '#include "frcnn_b200.h"', "int main(void) {", "    const void* fns[] = {"]
    src += ["        (const void*)&%s," % n for n in names]
    src += ["    };", '    printf("%d %d\\n", frcnn_version(), (int)(sizeof(fns) / sizeof(fns[0])));', "    return 0;", "}"]
    c = tmp_path / "abi.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "abi"
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-Wno-pedantic", "-I", os.path.join(root, "include"), str(c), "-o", str(exe),
                           "-L", libdir, "-lfrcnn_b200", "-Wl,-rpath," + libdir])
    out = subprocess.check_output([str(exe)]).decode().split()
    assert int(out[0]) >= 100 and int(out[1]) == len(names)
