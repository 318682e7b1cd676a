"""ctypes binding of libfrcnn_b200.so (the C ABI declared in include/frcnn_b200.h).

There is NO fallback: if the shared library is missing the import raises with build
instructions; if a call fails the Python wrapper raises FrcnnError with the library's message.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfrcnn_b200.so")

OK, ERR_ARG, ERR_CUDA, ERR_WORKSPACE = 0, -1, -2, -3
NMS_GE_DOUBLE, NMS_GT_FLOAT = 0, 1


class FrcnnError(RuntimeError):
    pass


c_void_p, c_int, c_long, c_size_t = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_size_t
c_double, c_float, c_char_p = ctypes.c_double, ctypes.c_float, ctypes.c_char_p

# name -> (restype, argtypes): mirrors include/frcnn_b200.h one to one.
SIGNATURES = {
    "frcnn_version": (c_int, []),
    "frcnn_last_error": (c_char_p, []),
    "_nms": (None, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_int]),
    "frcnn_cpu_nms_host": (c_int, [c_void_p, c_int, c_double, c_void_p, c_int]),
    "frcnn_host_nms_phase_cycles": (c_int, [c_void_p]),
    "frcnn_match_class_dets": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int]),
    "frcnn_nms_workspace_bytes": (c_size_t, [c_int]),
    "frcnn_nms": (c_int, [c_void_p, c_int, c_double, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_proposals_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "frcnn_proposals": (c_int, [c_void_p, c_long, c_long, c_int, c_void_p, c_long, c_long, c_void_p,
                                c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_double,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                c_void_p]),
    "frcnn_conv2d": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                             c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "frcnn_conv2d_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                   c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "frcnn_linear_batch_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "frcnn_linear_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                   c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    "frcnn_pack_image_c8_batch": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_long, c_long, c_long, c_long, c_void_p, c_void_p,
                                          c_void_p]),
    "frcnn_conv3x3_c8_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                       c_void_p, c_void_p, c_void_p]),
    "frcnn_linear_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "frcnn_linear": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                             c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    "frcnn_conv2d_set_tile": (None, [c_int, c_int, c_int]),
    "frcnn_conv2d_set_cta_group": (None, [c_int]),
    "frcnn_conv2d_set_max_ctas": (None, [c_int]),
    "frcnn_conv2d_set_smem_reserve": (None, [c_int]),
    "frcnn_conv2d_last_plan": (c_int, [c_void_p, c_int]),
    "frcnn_set_programmatic_launch": (None, [c_int]),
    "frcnn_host_alloc": (c_void_p, [c_size_t]),
    "frcnn_host_free": (c_int, [c_void_p]),
    "frcnn_memcpy_h2d_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_memcpy_d2h_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_stream_synchronize": (c_int, [c_void_p]),
    "frcnn_host_copy": (c_int, [c_void_p, c_void_p, c_size_t]),
    "frcnn_upload_pageable": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_pack_conv_weights": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                        c_int, c_int, c_int, c_void_p]),
    "frcnn_pack_image": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_preprocess_bgr8": (c_int, [c_void_p, c_int, c_int, c_double, c_double, c_double, c_double, c_int, c_int,
                                      c_void_p, c_void_p]),
    "frcnn_pack_image_im2col3x3": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_image_c8_elems": (c_size_t, [c_int, c_int]),
    "frcnn_pack_image_c8": (c_int, [c_void_p, c_int, c_int, c_int, c_long, c_long, c_long, c_void_p, c_void_p, c_void_p]),
    "frcnn_pack_conv_weights_c8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_conv3x3_c8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                 c_void_p]),
    "frcnn_pack_image_im2col3x3_strided": (c_int, [c_void_p, c_int, c_int, c_int, c_long, c_long, c_long, c_void_p, c_void_p, c_void_p]),
    "frcnn_pack_conv_weights_im2col3x3": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_unpack_nhwc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "frcnn_maxpool2x2_ceil": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_roi_pool": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                               c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_head_decode": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                  c_void_p, c_void_p, c_void_p]),
    "frcnn_bbox_decode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                  c_void_p]),
    "frcnn_bbox_overlaps": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "frcnn_anchor_targets_workspace_bytes": (c_size_t, [c_int, c_int]),
    "frcnn_anchor_targets": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_double,
                                     c_double, c_int, c_int, c_int, ctypes.c_ulonglong, c_void_p, c_int, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_rpn_loss_workspace_bytes": (c_size_t, [c_int]),
    "frcnn_rpn_loss": (c_int, [c_void_p, c_long, c_long, c_void_p, c_long, c_long, c_void_p, c_int, c_int, c_int, c_int,
                               c_int, c_int, c_void_p, c_void_p, c_void_p, c_double, c_double, c_double, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_anchor_targets_batch_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "frcnn_anchor_targets_batch": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int,
                                           c_void_p, c_double, c_double, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_rpn_loss_batch_workspace_bytes": (c_size_t, [c_int, c_int]),
    "frcnn_rpn_loss_batch": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_double, c_double, c_double, c_void_p, c_void_p, c_void_p,
                                     c_size_t, c_void_p]),
    "frcnn_grad_prepare_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                         c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "frcnn_gemm_nt_splitk_splits": (c_int, [c_int, c_int]),
    "frcnn_gemm_nt_splitk": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                     c_void_p, c_void_p, c_int, c_void_p]),
    "frcnn_padded_pixels": (c_long, [c_int, c_int, c_void_p]),
    "frcnn_grad_prepare": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                   c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "frcnn_maxpool3x3s2_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_grad_prepare_stride2": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_int, c_void_p]),
    "frcnn_maxpool3x3s2_backward_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                                  c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_grad_prepare_stride2_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                                 c_void_p, c_void_p, c_int, c_void_p]),
    "frcnn_fold_batchnorm": (c_int, [c_void_p, c_void_p, c_int, c_long, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_wgrad_reduce_scaled": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_wgrad_reduce": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "frcnn_bias_grad": (c_int, [c_void_p, c_void_p, c_int, c_long, c_float, c_void_p, c_void_p]),
    "frcnn_sgd_momentum": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_float, c_float, c_float, c_void_p]),
    "frcnn_cast_f32_bf16": (c_int, [c_void_p, c_void_p, c_long, c_void_p]),
    "frcnn_sgd_momentum_bf16g": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_float, c_float, c_float, c_void_p]),
    "frcnn_optimizer_update": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_long, c_void_p, c_void_p]),
    "frcnn_pack_conv_weights_dgrad": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_conv2d_res": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_pack_image_im2col": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_pack_conv_weights_im2col": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_maxpool3x3s2_ceil": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_subsample2x": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_pack_image_im2col_batch": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                              c_void_p]),
    "frcnn_pack_image_im2col_batch_ext": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                                  c_void_p, c_void_p, c_void_p]),
    "frcnn_maxpool3x3s2_ceil_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_maxpool3x3s2_ceil_batch_ext": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                                  c_void_p]),
    "frcnn_subsample2x_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_conv2d_res_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                       c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_conv2d_res_batch_ext": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                           c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "frcnn_resnet_level_extents": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "frcnn_preprocess_bgr8_canvas_im2col": (c_int, [c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                    c_int, c_double, c_double, c_double, c_int, c_int, c_int, c_int, c_void_p,
                                                    c_void_p, c_void_p]),
    "frcnn_preprocess_voc_canvas_im2col": (c_int, [c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                   c_int, c_double, c_double, c_double, c_int, c_int, c_int, c_int, c_void_p,
                                                   c_void_p, c_void_p]),
    "frcnn_voc_scale_gt_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_voc_augment_batch": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_preprocess_voc_canvas_im2col_flip": (c_int, [c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                        c_int, c_int, c_int, c_double, c_double, c_double, c_int, c_int, c_int, c_int,
                                                        c_void_p, c_void_p, c_void_p]),
    "frcnn_voc_flip_scale_gt_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                              c_void_p]),
    "frcnn_roi_overlaps": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_roi_targets": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_bbox_transform": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "frcnn_keep_inside": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "frcnn_rcnn_loss": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_double, c_double, c_void_p,
                                c_void_p, c_void_p]),
    "frcnn_dropout": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_float, c_void_p]),
    "frcnn_roi_pool_backward_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "frcnn_roi_pool_backward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_float,
                                        c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "frcnn_proposal_targets_batch": (c_int, [c_int, c_void_p, c_long, c_void_p, c_long, c_int, c_void_p, c_int, c_void_p, c_int,
                                             c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_rcnn_loss_batch": (c_int, [c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_double,
                                      c_double, c_void_p, c_void_p, c_void_p]),
    "frcnn_roi_pool_backward_batch_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "frcnn_roi_pool_backward_batch_ext": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_long, c_void_p, c_long,
                                                  c_int, c_int, c_int, c_float, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                                  c_void_p, c_size_t, c_void_p]),
    "frcnn_dropout_masks_batch": (c_int, [c_int, c_int, c_int, c_void_p, ctypes.c_ulonglong, c_void_p, c_void_p]),
    "frcnn_forward_workspace_bytes": (c_size_t, [c_void_p]),
    "frcnn_forward_vgg16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p,
                                    c_void_p]),
    "frcnn_debug_sort_clocks": (None, [c_void_p]),
    "frcnn_proposals_batch_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "frcnn_proposals_batch": (c_int, [c_int, c_void_p, c_long, c_long, c_long, c_int, c_void_p, c_long, c_long, c_long, c_void_p,
                                      c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_double,
                                      c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p, c_long,
                                      c_void_p, c_long, c_void_p, c_size_t, c_void_p]),
    "frcnn_maxpool2x2_ceil_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frcnn_roi_pool_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_long, c_void_p, c_long, c_int, c_int,
                                     c_int, c_float, c_void_p, c_void_p, c_void_p, c_long, c_void_p]),
    "frcnn_head_decode_batch": (c_int, [c_int, c_void_p, c_void_p, c_int, c_long, c_void_p, c_long, c_void_p, c_long, c_int, c_int,
                                        c_int, c_int, c_void_p, c_long, c_void_p, c_long, c_void_p]),
    "frcnn_detect_batch": (c_int, [c_int, c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_int, c_int, c_double, c_float,
                                   c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p]),
    "frcnn_forward_batch_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "frcnn_forward_vgg16_batch": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p,
                                          c_void_p, c_void_p]),
    "frcnn_proposals_batch_ext": (c_int, [c_int, c_void_p, c_long, c_long, c_long, c_int, c_void_p, c_long, c_long, c_long, c_void_p,
                                          c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_double,
                                          c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p, c_size_t, c_void_p]),
    "frcnn_conv2d_batch_ext": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                       c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "frcnn_pack_image_c8_batch_ext": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_long, c_long, c_long, c_long, c_void_p,
                                              c_void_p, c_void_p, c_void_p]),
    "frcnn_preprocess_bgr8_canvas": (c_int, [c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                             c_double, c_double, c_double, c_void_p, c_void_p, c_void_p]),
    "frcnn_conv3x3_c8_batch_ext": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                           c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_roi_pool_batch_ext": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_long, c_void_p, c_long, c_int,
                                         c_int, c_int, c_float, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_long, c_void_p]),
    "frcnn_head_decode_batch_ext": (c_int, [c_int, c_void_p, c_void_p, c_int, c_long, c_void_p, c_long, c_void_p, c_long, c_int,
                                            c_int, c_void_p, c_void_p, c_long, c_void_p, c_long, c_void_p]),
    "frcnn_detect": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_double, c_float, c_void_p, c_void_p,
                             c_void_p, c_void_p]),
    "frcnn_detection_lists_batch": (c_int, [c_int, c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p,
                                            c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frcnn_voc_eval_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "frcnn_voc_eval_append_batch": (c_int, [c_int, c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p, c_long, c_void_p,
                                            c_int, c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "frcnn_voc_eval": (c_int, [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_double, c_void_p,
                               c_void_p, c_size_t, c_void_p]),
    "frcnn_forward_vgg16_canvas_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "frcnn_forward_vgg16_canvas": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p,
                                           c_void_p, c_void_p, c_void_p]),
    "frcnn_raw_header_bytes": (c_size_t, [c_int]),
    "frcnn_detect_vgg16_raw": (c_int, [c_void_p, c_void_p, c_int, c_void_p, ctypes.c_longlong, c_double, c_double, c_double, c_void_p,
                                       c_double, c_float, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p]),
}

_lib = None


def load():
    """dlopen the library and attach prototypes (works on a CPU-only box: no libcuda dependency)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FrcnnError(
            "libfrcnn_b200.so not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C chainer-faster-rcnn_b200/csrc` (needs nvcc; there is no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


_pylib = None


def load_gil():
    """A second handle on the same library whose calls KEEP the GIL (ctypes.PyDLL): for sub-microsecond pure-host helpers,
    where releasing and re-acquiring the GIL (a condition-variable round trip under several caller threads) would cost
    a hundred times the call."""
    global _pylib
    if _pylib is None:
        load()
        lib = ctypes.PyDLL(LIB_PATH)
        fn = lib.frcnn_match_class_dets
        fn.restype, fn.argtypes = SIGNATURES["frcnn_match_class_dets"]
        _pylib = lib
    return _pylib


def last_error():
    msg = load().frcnn_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(status, what):
    if status != OK:
        raise FrcnnError("%s failed (status %d): %s" % (what, status, last_error()))


# ---- the structs of the whole-graph entry (include/frcnn_b200.h: frcnn_forward_config / frcnn_packed_layer / frcnn_vgg16_weights)
class ForwardConfig(ctypes.Structure):
    _fields_ = [("H", c_int), ("W", c_int), ("num_classes", c_int), ("n_anchors", c_int), ("feat_stride", c_int),
                ("pre_nms_top_n", c_int), ("post_nms_top_n", c_int), ("min_size", c_int), ("nms_thresh", c_double), ("x3", c_int)]


class PackedLayer(ctypes.Structure):
    _fields_ = [("hi", c_void_p), ("lo", c_void_p), ("bias", c_void_p)]


class Vgg16Weights(ctypes.Structure):
    _fields_ = [("conv", PackedLayer * 13), ("rpn3", PackedLayer), ("rpn_heads", PackedLayer), ("fc6", PackedLayer),
                ("fc7", PackedLayer), ("head", PackedLayer), ("anchors", c_void_p)]
