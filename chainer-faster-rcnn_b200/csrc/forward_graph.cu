// forward_graph.cu -- frcnn_forward_vgg16(_batch / _canvas) and frcnn_detect_vgg16_raw: the whole forward detection path of
// one image, of N same-size images, or of N images of different sizes on a canvas, behind ONE C-ABI call.
//
// FasterRCNN.__call__, inference branch (/root/reference models/faster_rcnn.py:92-134,175-178): trunk (models/vgg16.py:38-82)
// -> RPN (models/region_proposal_network.py:117-124) -> ProposalLayer (models/proposal_layer.py:102-198) -> RoI pooling ->
// fc6 / fc7 -> cls_score | bbox_pred -> softmax + decode + clip.  This is pure host orchestration: it carves the caller's
// workspace and enqueues the same kernels, in the same order, as frcnn_b200/engine.py's BatchPlan / CanvasBatchPlan -- for
// callers that have no Python (the launch sequence is static, so the caller may capture it into a CUDA graph).  No allocation,
// no synchronisation.  One image is the batch of N = 1; every stage is one launch for all N images.
#include "common.cuh"

using namespace frcnn;

namespace {

struct Plane { void *hi, *lo; };

struct Carver {
    char* base;
    size_t off;
    bool x3;
    void* take(size_t bytes) {
        void* p = base ? base + off : nullptr;
        off += align_up(bytes, 256);
        return p;
    }
    Plane act(long elems) {
        Plane p;
        p.hi = take((size_t)elems * 2);
        p.lo = x3 ? take((size_t)elems * 2) : nullptr;
        return p;
    }
};

// VGG16 trunk table (models/vgg16.py:38-69): {Cin, Cout, pool after}
const int kVgg[13][3] = {{3, 64, 0},    {64, 64, 1},   {64, 128, 0},  {128, 128, 1}, {128, 256, 0}, {256, 256, 0}, {256, 256, 1},
                         {256, 512, 0}, {512, 512, 0}, {512, 512, 1}, {512, 512, 0}, {512, 512, 0}, {512, 512, 0}};

struct Layout {
    Plane x_col, act[13], rpn_mid, pool5, fc6, fc7;
    float *rpn_out, *head_out, *rois, *scores;
    void *prop_ws, *fc_ws;
    size_t prop_ws_bytes, fc_ws_bytes;
    int *keep_idx, *keep_count, *conf_count;    // the per-class NMS lists of frcnn_detect_vgg16_raw (canvas workspace only)
    int fh, fw, rpn_ld, head_ld, ld1;
    size_t total;
};

int round32(int v) { return (v + 31) / 32 * 32; }

// The workspace of N images: every activation is [N][...] (image n's block right after image n-1's), the head
// activations hold ld1 = round_up(post_nms_top_n, 32) rows per image (frcnn_linear_batch's segments).  The canvas workspace
// (lists = true) appends frcnn_detect_batch's outputs, [N][num_classes-1][post_nms_top_n] keep_idx and [N][num_classes-1]
// keep_count / conf_count; everything before them is the same-size layout of config->H x config->W.
Layout carve(const frcnn_forward_config& c, int N, void* workspace, bool lists = false) {
    Layout L;
    Carver k{(char*)workspace, 0, c.x3 != 0};
    L.x_col = k.act((long)N * frcnn_image_c8_elems(c.H, c.W));    // compact first-layer input [N][H][W+2][8]
    int h = c.H, w = c.W;
    for (int i = 0; i < 13; ++i) {
        if (kVgg[i][2]) { h = (h + 1) / 2; w = (w + 1) / 2; }          // the pool is fused into this conv's epilogue
        L.act[i] = k.act((long)N * h * w * kVgg[i][1]);
    }
    L.fh = h; L.fw = w;
    L.rpn_ld = round32(6 * c.n_anchors);
    L.head_ld = round32(5 * c.num_classes);
    L.ld1 = round32(c.post_nms_top_n);
    const long rows = (long)N * L.ld1;
    L.rpn_mid = k.act((long)N * h * w * 512);
    L.rpn_out = (float*)k.take((size_t)N * h * w * L.rpn_ld * 4);
    L.prop_ws_bytes = frcnn_proposals_batch_workspace_bytes(N, c.n_anchors, h, w, c.pre_nms_top_n);
    L.prop_ws = k.take(L.prop_ws_bytes);
    L.rois = (float*)k.take((size_t)N * c.post_nms_top_n * 4 * 4);
    L.scores = (float*)k.take((size_t)N * c.post_nms_top_n * 4);
    L.pool5 = k.act(rows * 49 * 512);
    L.fc6 = k.act(rows * 4096);
    L.fc7 = k.act(rows * 4096);
    L.head_out = (float*)k.take((size_t)rows * L.head_ld * 4);
    L.fc_ws_bytes = frcnn_linear_batch_workspace_bytes(N, c.post_nms_top_n, 49 * 512, 4096);
    const size_t b7 = frcnn_linear_batch_workspace_bytes(N, c.post_nms_top_n, 4096, 4096);
    const size_t bh = frcnn_linear_batch_workspace_bytes(N, c.post_nms_top_n, 4096, 5 * c.num_classes);
    if (b7 > L.fc_ws_bytes) L.fc_ws_bytes = b7;
    if (bh > L.fc_ws_bytes) L.fc_ws_bytes = bh;
    L.fc_ws = k.take(L.fc_ws_bytes);
    L.keep_idx = L.keep_count = L.conf_count = nullptr;
    if (lists) {
        const long nc1 = (long)N * (c.num_classes - 1);
        L.keep_idx = (int*)k.take((size_t)nc1 * c.post_nms_top_n * 4);
        L.keep_count = (int*)k.take((size_t)nc1 * 4);
        L.conf_count = (int*)k.take((size_t)nc1 * 4);
    }
    L.total = k.off;
    return L;
}

int check_config(const frcnn_forward_config* c) {
    FRCNN_REQUIRE(c != nullptr, "frcnn_forward: null config");
    FRCNN_REQUIRE(c->H >= 16 && c->W >= 16, "frcnn_forward: image %dx%d too small (one feature cell needs 16x16)", c->H, c->W);
    FRCNN_REQUIRE(c->num_classes >= 2 && c->n_anchors >= 1 && c->feat_stride == 16, "frcnn_forward: VGG16 trunk has feat_stride 16");
    FRCNN_REQUIRE(c->pre_nms_top_n > 0 && c->post_nms_top_n > 0 && c->post_nms_top_n <= 2048, "frcnn_forward: bad top-N limits");
    return FRCNN_OK;
}

int check_batch(int N) {
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "frcnn_forward: N must be in [1,65535] (got %d)", N);
    return FRCNN_OK;
}

// The checks every entry makes before it enqueues anything, then the carve.  `inputs` is false when the entry's own input
// pointers are missing.
int begin(const frcnn_forward_config* config, const frcnn_vgg16_weights* wts, int N, bool inputs, void* workspace,
          size_t workspace_bytes, bool lists, float* out_prob, float* out_boxes, int* out_count, Layout& L) {
    int rc = check_config(config);
    if (rc != FRCNN_OK) return rc;
    if ((rc = check_batch(N)) != FRCNN_OK) return rc;
    FRCNN_REQUIRE(wts && inputs && workspace && out_prob && out_boxes && out_count, "frcnn_forward: null pointer");
    L = carve(*config, N, workspace, lists);
    if (workspace_bytes < L.total) {
        set_error("frcnn_forward: workspace %zu < %zu bytes", workspace_bytes, L.total);
        return FRCNN_ERR_WORKSPACE;
    }
    const bool x3 = config->x3 != 0;
    for (int i = 0; i < 13; ++i)
        FRCNN_REQUIRE(wts->conv[i].hi && wts->conv[i].bias && (!x3 || wts->conv[i].lo), "frcnn_forward: trunk layer %d weights missing", i);
    return FRCNN_OK;
}

// Where the images' sizes come from.  extents == NULL: N images of config->H x config->W that one clip bound (im_h, im_w)
// serves (the same-size launches).  Otherwise a canvas batch: device int32 [N][2] image sizes and clip bounds read at run
// time, and every stage that depends on them is the matching *_ext entry (CanvasBatchPlan).
struct Sizes {
    const int* extents;
    const int* im_info;
    int im_h, im_w;
};

// Everything after the first-layer pack, which has written L.x_col: trunk, RPN, ProposalLayer, RoI pooling and the head.
int forward_packed(const frcnn_forward_config& c, const frcnn_vgg16_weights* wts, int N, const Layout& L, const Sizes& sz,
                   float* out_prob, float* out_boxes, int* out_count, cudaStream_t stream) {
    const int* ext = sz.extents;
    int rc;
    // ---- trunk: conv1_1 as a K = 3 x 32 GEMM over the compact images (sliding-window tensor map), then 12 shared-halo 3x3 convs
    Plane x = L.x_col;
    int h = c.H, w = c.W, cin = 32, k = 0;      // k: 2x2 pools before the current layer (a canvas extent is ceil(extent / 2^k))
    for (int i = 0; i < 13; ++i) {
        const frcnn_packed_layer& l = wts->conv[i];
        if (i == 0 && ext)
            rc = frcnn_conv3x3_c8_batch_ext(x.hi, x.lo, N, h, w, l.hi, l.lo, l.bias, kVgg[0][1], 1, ext, L.act[0].hi, L.act[0].lo,
                                            stream);
        else if (i == 0)
            rc = frcnn_conv3x3_c8_batch(x.hi, x.lo, N, h, w, l.hi, l.lo, l.bias, kVgg[0][1], 1, L.act[0].hi, L.act[0].lo, stream);
        else if (ext)
            rc = frcnn_conv2d_batch_ext(x.hi, x.lo, N, h, w, cin, l.hi, l.lo, l.bias, kVgg[i][1], 3, 1, kVgg[i][2], L.act[i].hi,
                                        L.act[i].lo, nullptr, 0, ext, k, stream);
        else
            rc = frcnn_conv2d_batch(x.hi, x.lo, N, h, w, cin, l.hi, l.lo, l.bias, kVgg[i][1], 3, 1, kVgg[i][2], L.act[i].hi, L.act[i].lo,
                                    nullptr, 0, stream);
        if (rc != FRCNN_OK) return rc;
        if (kVgg[i][2]) { h = (h + 1) / 2; w = (w + 1) / 2; ++k; }
        x = L.act[i];
        cin = kVgg[i][1];
    }
    const Plane feat = x;
    // ---- RPN: 3x3 conv + ReLU, the merged twin 1x1 heads (fp32 [N*H*W, rpn_ld]), ProposalLayer with the 2A-way softmax fused
    if (ext) {
        if ((rc = frcnn_conv2d_batch_ext(feat.hi, feat.lo, N, h, w, 512, wts->rpn3.hi, wts->rpn3.lo, wts->rpn3.bias, 512, 3, 1, 0,
                                         L.rpn_mid.hi, L.rpn_mid.lo, nullptr, 0, ext, k, stream)) != FRCNN_OK) return rc;
        if ((rc = frcnn_conv2d_batch_ext(L.rpn_mid.hi, L.rpn_mid.lo, N, h, w, 512, wts->rpn_heads.hi, wts->rpn_heads.lo,
                                         wts->rpn_heads.bias, 6 * c.n_anchors, 1, 0, 0, nullptr, nullptr, L.rpn_out, L.rpn_ld, ext, k,
                                         stream)) != FRCNN_OK) return rc;
    } else {
        if ((rc = frcnn_conv2d_batch(feat.hi, feat.lo, N, h, w, 512, wts->rpn3.hi, wts->rpn3.lo, wts->rpn3.bias, 512, 3, 1, 0,
                                     L.rpn_mid.hi, L.rpn_mid.lo, nullptr, 0, stream)) != FRCNN_OK) return rc;
        if ((rc = frcnn_conv2d_batch(L.rpn_mid.hi, L.rpn_mid.lo, N, h, w, 512, wts->rpn_heads.hi, wts->rpn_heads.lo, wts->rpn_heads.bias,
                                     6 * c.n_anchors, 1, 0, 0, nullptr, nullptr, L.rpn_out, L.rpn_ld, stream)) != FRCNN_OK) return rc;
    }
    const int R = c.post_nms_top_n, NC = c.num_classes;
    const long rpn_is = (long)h * w * L.rpn_ld;
    if (ext)
        rc = frcnn_proposals_batch_ext(N, L.rpn_out, 1, L.rpn_ld, rpn_is, 1, L.rpn_out + 2 * c.n_anchors, 1, L.rpn_ld, rpn_is,
                                       wts->anchors, c.n_anchors, h, w, c.feat_stride, ext, k, sz.im_info, c.min_size, c.pre_nms_top_n,
                                       R, c.nms_thresh, L.rois, 4l * R, L.scores, R, out_count, 1, L.prop_ws, L.prop_ws_bytes, stream);
    else
        rc = frcnn_proposals_batch(N, L.rpn_out, 1, L.rpn_ld, rpn_is, 1, L.rpn_out + 2 * c.n_anchors, 1, L.rpn_ld, rpn_is, wts->anchors,
                                   c.n_anchors, h, w, c.feat_stride, sz.im_h, sz.im_w, c.min_size, c.pre_nms_top_n, R, c.nms_thresh,
                                   L.rois, 4l * R, L.scores, R, out_count, 1, nullptr, 0, nullptr, 0, nullptr, 0, L.prop_ws,
                                   L.prop_ws_bytes, stream);
    if (rc != FRCNN_OK) return rc;
    // ---- RoI pooling + head (rows past out_count[n] are zero)
    const float scale = 1.0f / (float)c.feat_stride;
    const long pool_is = (long)L.ld1 * 49 * 512;
    if (ext)
        rc = frcnn_roi_pool_batch_ext(feat.hi, feat.lo, N, h, w, 512, L.rois, 4l * R, out_count, 1, R, 7, 7, scale, ext, k, L.pool5.hi,
                                      L.pool5.lo, nullptr, pool_is, stream);
    else
        rc = frcnn_roi_pool_batch(feat.hi, feat.lo, N, h, w, 512, L.rois, 4l * R, out_count, 1, R, 7, 7, scale, L.pool5.hi, L.pool5.lo,
                                  nullptr, pool_is, stream);
    if (rc != FRCNN_OK) return rc;
    if ((rc = frcnn_linear_batch(L.pool5.hi, L.pool5.lo, N, R, 49 * 512, wts->fc6.hi, wts->fc6.lo, wts->fc6.bias, 4096, 1, out_count, 1,
                                 L.fc6.hi, L.fc6.lo, nullptr, 0, L.fc_ws, L.fc_ws_bytes, stream)) != FRCNN_OK) return rc;
    if ((rc = frcnn_linear_batch(L.fc6.hi, L.fc6.lo, N, R, 4096, wts->fc7.hi, wts->fc7.lo, wts->fc7.bias, 4096, 1, out_count, 1, L.fc7.hi,
                                 L.fc7.lo, nullptr, 0, L.fc_ws, L.fc_ws_bytes, stream)) != FRCNN_OK) return rc;
    if ((rc = frcnn_linear_batch(L.fc7.hi, L.fc7.lo, N, R, 4096, wts->head.hi, wts->head.lo, wts->head.bias, 5 * NC, 0, out_count, 1,
                                 nullptr, nullptr, L.head_out, L.head_ld, L.fc_ws, L.fc_ws_bytes, stream)) != FRCNN_OK) return rc;
    const long head_is = (long)L.ld1 * L.head_ld;
    if (ext)
        return frcnn_head_decode_batch_ext(N, L.head_out, L.head_out + NC, L.head_ld, head_is, L.rois, 4l * R, out_count, 1, R, NC,
                                           sz.im_info, out_prob, (long)R * NC, out_boxes, 4l * R * NC, stream);
    return frcnn_head_decode_batch(N, L.head_out, L.head_out + NC, L.head_ld, head_is, L.rois, 4l * R, out_count, 1, R, NC, sz.im_h,
                                   sz.im_w, out_prob, (long)R * NC, out_boxes, 4l * R * NC, stream);
}

// The forward path over N images of one shape: every stage is one launch sequence for the whole batch.
int forward_n(const frcnn_forward_config* config, const frcnn_vgg16_weights* wts, int N, const float* images_nchw, int im_h,
              int im_w, void* workspace, size_t workspace_bytes, float* out_prob, float* out_boxes, int* out_count,
              cudaStream_t stream) {
    Layout L;
    int rc = begin(config, wts, N, images_nchw != nullptr, workspace, workspace_bytes, false, out_prob, out_boxes, out_count, L);
    if (rc != FRCNN_OK) return rc;
    const frcnn_forward_config& c = *config;
    const long hw = (long)c.H * c.W;
    if ((rc = frcnn_pack_image_c8_batch(images_nchw, N, 3, c.H, c.W, 3 * hw, hw, c.W, 1, L.x_col.hi, L.x_col.lo, stream)) != FRCNN_OK)
        return rc;
    const Sizes sz = {nullptr, nullptr, im_h, im_w};
    return forward_packed(c, wts, N, L, sz, out_prob, out_boxes, out_count, stream);
}

// The raw block [header | pixels] of frcnn_detect_vgg16_raw: field f of the header starts 8 * N * f bytes in.
const void* raw_field(const void* block, int N, int f) { return (const char*)block + 8l * N * f; }

}  // namespace

extern "C" {

size_t frcnn_forward_workspace_bytes(const frcnn_forward_config* config) {
    FRCNN_ENTRY();
    if (check_config(config) != FRCNN_OK) return 0;
    return carve(*config, 1, nullptr).total;
}

size_t frcnn_forward_batch_workspace_bytes(const frcnn_forward_config* config, int N) {
    FRCNN_ENTRY();
    if (check_config(config) != FRCNN_OK || check_batch(N) != FRCNN_OK) return 0;
    return carve(*config, N, nullptr).total;
}

int frcnn_forward_vgg16(const frcnn_forward_config* config, const frcnn_vgg16_weights* wts, const float* image_chw, int im_h,
                        int im_w, void* workspace, size_t workspace_bytes, float* out_prob, float* out_boxes, int* out_count,
                        void* stream) {
    FRCNN_ENTRY();
    return forward_n(config, wts, 1, image_chw, im_h, im_w, workspace, workspace_bytes, out_prob, out_boxes, out_count,
                     static_cast<cudaStream_t>(stream));
}

int frcnn_forward_vgg16_batch(const frcnn_forward_config* config, const frcnn_vgg16_weights* wts, int N, const float* images_nchw,
                              int im_h, int im_w, void* workspace, size_t workspace_bytes, float* out_prob, float* out_boxes,
                              int* out_count, void* stream) {
    FRCNN_ENTRY();
    return forward_n(config, wts, N, images_nchw, im_h, im_w, workspace, workspace_bytes, out_prob, out_boxes, out_count,
                     static_cast<cudaStream_t>(stream));
}

size_t frcnn_forward_vgg16_canvas_workspace_bytes(const frcnn_forward_config* config, int N) {
    FRCNN_ENTRY();
    if (check_config(config) != FRCNN_OK || check_batch(N) != FRCNN_OK) return 0;
    return carve(*config, N, nullptr, true).total;
}

int frcnn_forward_vgg16_canvas(const frcnn_forward_config* config, const frcnn_vgg16_weights* wts, int N, const float* images_nchw,
                               const int* extents, const int* im_info, void* workspace, size_t workspace_bytes, float* out_prob,
                               float* out_boxes, int* out_count, void* stream) {
    FRCNN_ENTRY();
    Layout L;
    int rc = begin(config, wts, N, images_nchw && extents && im_info, workspace, workspace_bytes, true, out_prob, out_boxes, out_count,
                   L);
    if (rc != FRCNN_OK) return rc;
    const frcnn_forward_config& c = *config;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long hw = (long)c.H * c.W;
    if ((rc = frcnn_pack_image_c8_batch_ext(images_nchw, N, 3, c.H, c.W, 3 * hw, hw, c.W, 1, extents, L.x_col.hi, L.x_col.lo, st)) !=
        FRCNN_OK)
        return rc;
    const Sizes sz = {extents, im_info, 0, 0};
    return forward_packed(c, wts, N, L, sz, out_prob, out_boxes, out_count, st);
}

size_t frcnn_raw_header_bytes(int N) {
    FRCNN_ENTRY();
    if (check_batch(N) != FRCNN_OK) return 0;
    return align_up((size_t)8 * N * FRCNN_RAW_FIELDS, 256);
}

int frcnn_detect_vgg16_raw(const frcnn_forward_config* config, const frcnn_vgg16_weights* wts, int N, const void* block,
                           long long arena_bytes, double mean_b, double mean_g, double mean_r, const double* im_scale,
                           double det_nms_thresh, float det_conf, void* workspace, size_t workspace_bytes, float* out_prob,
                           float* out_boxes, int* out_count, int* out_dets, float* out_scores, int* out_det_count, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(arena_bytes > 0, "frcnn_detect_vgg16_raw: arena_bytes must be positive (got %lld)", arena_bytes);
    FRCNN_REQUIRE(((uintptr_t)block & 7) == 0, "frcnn_detect_vgg16_raw: the block must be 8-byte aligned");
    Layout L;
    int rc = begin(config, wts, N, block && im_scale && out_dets && out_scores && out_det_count, workspace, workspace_bytes, true,
                   out_prob, out_boxes, out_count, L);
    if (rc != FRCNN_OK) return rc;
    const frcnn_forward_config& c = *config;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int* extents = (const int*)raw_field(block, N, FRCNN_RAW_EXTENTS);
    const Sizes sz = {extents, (const int*)raw_field(block, N, FRCNN_RAW_IM_INFO), 0, 0};
    const unsigned char* arena = (const unsigned char*)block + frcnn_raw_header_bytes(N);
    if ((rc = frcnn_preprocess_bgr8_canvas(arena, arena_bytes, (const long long*)raw_field(block, N, FRCNN_RAW_SRC_OFF),
                                           (const int*)raw_field(block, N, FRCNN_RAW_SRC_HW),
                                           (const double*)raw_field(block, N, FRCNN_RAW_INV_SCALE), extents, N, c.H, c.W, mean_b,
                                           mean_g, mean_r, L.x_col.hi, L.x_col.lo, st)) != FRCNN_OK)
        return rc;
    if ((rc = forward_packed(c, wts, N, L, sz, out_prob, out_boxes, out_count, st)) != FRCNN_OK) return rc;
    const int R = c.post_nms_top_n, NC = c.num_classes;
    if ((rc = frcnn_detect_batch(N, out_prob, (long)R * NC, out_boxes, 4l * R * NC, out_count, 1, R, NC, det_nms_thresh, det_conf,
                                 L.keep_idx, (long)(NC - 1) * R, L.keep_count, NC - 1, L.conf_count, NC - 1, st)) != FRCNN_OK)
        return rc;
    return frcnn_detection_lists_batch(N, out_prob, (long)R * NC, out_boxes, 4l * R * NC, L.keep_idx, (long)(NC - 1) * R, L.conf_count,
                                       NC - 1, im_scale, R, NC, out_dets, out_scores, out_det_count, st);
}

}  // extern "C"
