"""CPU tests of the canvas-batch C entries (the *_batch_ext functions of include/frcnn_b200.h): a NULL extents or clip
array, a bad image count or a bad halving count is rejected with FRCNN_ERR_ARG and a message before anything touches the
device, so these run without a GPU."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


P = ctypes.c_void_p(256)            # never dereferenced: every call below fails its argument checks first


def _arg_error(status, words):
    from frcnn_b200 import _lib
    msg = _lib.last_error()
    return status == _lib.ERR_ARG and all(w in msg for w in words)


def test_conv_entries_need_extents(lib):
    assert _arg_error(lib.frcnn_conv2d_batch_ext(P, None, 2, 8, 8, 64, P, None, P, 64, 3, 1, 0, P, None, None, 0, None, 0, None),
                      ["extents"])
    assert _arg_error(lib.frcnn_conv2d_batch_ext(P, None, 0, 8, 8, 64, P, None, P, 64, 3, 1, 0, P, None, None, 0, P, 0, None),
                      ["N >= 1"])
    for bad in (-1, 31):
        assert _arg_error(lib.frcnn_conv2d_batch_ext(P, None, 2, 8, 8, 64, P, None, P, 64, 3, 1, 0, P, None, None, 0, P, bad, None),
                          ["halvings"])
    assert _arg_error(lib.frcnn_conv3x3_c8_batch_ext(P, None, 2, 8, 8, P, None, P, 64, 1, None, P, None, None), ["extents"])
    assert _arg_error(lib.frcnn_conv3x3_c8_batch_ext(P, None, 0, 8, 8, P, None, P, 64, 1, P, P, None, None), ["N=0"])
    assert _arg_error(lib.frcnn_pack_image_c8_batch_ext(P, 2, 3, 8, 8, 192, 64, 8, 1, None, P, None, None), ["extents"])
    assert _arg_error(lib.frcnn_pack_image_c8_batch_ext(P, 0, 3, 8, 8, 192, 64, 8, 1, P, P, None, None), ["N=0"])


def test_post_processing_entries_need_extents_and_clips(lib):
    f1 = ctypes.c_float(1.0 / 16)
    assert _arg_error(lib.frcnn_roi_pool_batch_ext(P, None, 2, 8, 8, 64, P, 4 * 300, None, 0, 300, 7, 7, f1, None, 4, P, None,
                                                   None, 300 * 49 * 64, None), ["extents"])
    assert _arg_error(lib.frcnn_roi_pool_batch_ext(P, None, 0, 8, 8, 64, P, 4 * 300, None, 0, 300, 7, 7, f1, P, 4, P, None,
                                                   None, 300 * 49 * 64, None), ["N must be"])
    assert _arg_error(lib.frcnn_roi_pool_batch_ext(P, None, 2, 8, 8, 64, P, 4 * 300, None, 0, 300, 7, 7, f1, P, 40, P, None,
                                                   None, 300 * 49 * 64, None), ["halvings"])
    assert _arg_error(lib.frcnn_head_decode_batch_ext(2, P, P, 128, 300 * 128, P, 1200, None, 0, 300, 21, None, P, 6300, P, 25200,
                                                      None), ["im_info"])
    assert _arg_error(lib.frcnn_head_decode_batch_ext(70000, P, P, 128, 300 * 128, P, 1200, None, 0, 300, 21, P, P, 6300, P,
                                                      25200, None), ["N must be"])
    for n, ext, info, words in ((2, None, P, ["extents"]), (2, P, None, ["im_info"]), (0, P, P, ["N must be"])):
        assert _arg_error(lib.frcnn_proposals_batch_ext(n, P, 1, 64, 64 * 64, 1, P, 1, 64, 64 * 64, P, 9, 8, 8, 16, ext, 4, info, 16,
                                                        6000, 300, 0.7, P, 1200, P, 300, P, 1, P, 1 << 30, None), words)
    assert _arg_error(lib.frcnn_proposals_batch_ext(2, P, 1, 64, 64 * 64, 1, P, 1, 64, 64 * 64, P, 9, 8, 8, 16, P, 31, P, 16,
                                                    6000, 300, 0.7, P, 1200, P, 300, P, 1, P, 1 << 30, None), ["halvings"])
