"""The reference's two training steps on the device.

RpnTrainer -- one train_rpn.py step: forward (trunk + RPN) -> AnchorTargetLayer -> rpn_loss -> backward through the RPN
heads, the RPN 3x3 conv and the 13 trunk convs -> [gradient all-reduce] -> WeightDecay + the optimizer's rule
(MomentumSGD by default; Adam, AdaGrad or RMSprop through `optimizer=`, frcnn_b200.optimizers).
RcnnTrainer -- one train_rcnn.py step: trunk -> frozen test-mode RPN -> ProposalTargetLayer -> RoI pool -> fc6/fc7 with
dropout -> head losses -> backward through the head, the RoI pooling and the trunk -> the same optimizer.
CanvasRpnTrainer -- RpnTrainer's step on N images of different sizes per update (an N-slot canvas), one captured graph.
CanvasRcnnTrainer -- RcnnTrainer's step on such a canvas, with device-side RoI sampling and dropout masks.
JointTrainer -- approximate joint training (py-faster-rcnn's end2end): one trunk forward, the trained RPN once, rpn_loss and
ProposalLayer from its output, RcnnTrainer's head and loss_rcnn; one backward of rpn_loss + loss_rcnn, the feature map's two
gradients joined in the epilogue of the RPN conv's data gradient; one update of every parameter.
CanvasJointTrainer -- JointTrainer's step on a canvas, one captured graph.

Every trainer, here and in resnet_train, is one trunk (_Vgg16Trunk, _ResNetTrunk: layers, forward, backward from the
feature map's gradient, repacking) and one step (_RpnStep, _RcnnStep, _JointStep, or on a canvas _CanvasRpnStep,
_CanvasRcnnStep, _CanvasJointStep), all launching through _ConvTrainer's launch layer over one image, which _CanvasSteps
overrides for a canvas.  _JointStep runs the RPN and RCNN steps' own halves (forward after the trunk, backward down to the
feature map's gradient).

Mirrors /root/reference train_rpn.py:144-179 with `model.rpn_train = True`: FasterRCNN.__call__ takes the RPN training
branch (models/faster_rcnn.py:114-116 -> models/region_proposal_network.py:117-156), the optimizer is
MomentumSGD(lr=0.001) (momentum 0.9 default) + WeightDecay(0.0005) (train_rpn.py:165-167).  Only parameters that receive a
gradient are updated (Chainer v1 `cleargrads`: fc6/fc7/cls_score/bbox_pred have grad None in RPN mode and are skipped).

Every dense contraction runs on the tcgen05 kernel of the forward path:
    forward conv     frcnn_conv2d                       (pools NOT fused here: backward needs the un-pooled maps)
    data gradient    frcnn_conv2d with the 180-degree rotated, in/out-swapped filter (frcnn_pack_conv_weights_dgrad)
    weight gradient  frcnn_gemm_nt_splitk over the zero-padded pixel axis (9 tap groups x K splits), reduced in fixed order
and the element-wise backward ops (ReLU mask, max-pool routing, hi/lo split, transposition) are fused into
frcnn_grad_prepare.  Gradients / master weights / momentum are float32 in three flat buffers (one NCCL all-reduce).
"""
import numpy as np
import torch

from . import ops, optimizers, preprocess, shard, train_ops
from ._lib import FrcnnError
from .engine import ImageInput, RawPhotoInput, vgg16_schedule

ROIS_PER_IMAGE, FG_FRACTION = 128, 0.25                          # models/proposal_target_layer.py:49-50
FG_THRESH, BG_THRESH_HI, BG_THRESH_LO = 0.5, 0.5, 0.1            # :46-48
_STEPS = vgg16_schedule(1, 1, fuse_pool=False)[0]                # the layer table; training never fuses a pool
TRUNK = [s[:3] for s in _STEPS]                                  # (name, cin, cout) x 13
POOL_AFTER = {s.name for s in _STEPS if s.pool_after}


def _entries(layers, params):
    """[(name, shape)] in flat-buffer order: W, then b unless the layer has bias=False, of every layer in `layers`, then
    `params` in the given order."""
    out = []
    for L in layers:
        out.append((L["name"] + "/W", (L["cout"], L["cin"], L["k"], L["k"])))
        if L.get("bias", True):
            out.append((L["name"] + "/b", (L["cout"],)))
    return out + [(n, tuple(sh)) for n, sh in params]


def _fc6_to_hwc(name, a):                           # fc6 columns (c, h, w) -> (h, w, c), the order the RoI pooling emits
    return a.reshape(4096, -1, 49).transpose(0, 2, 1) if name == "fc6/W" else a


class _ConvTrainer(object):
    """Shared by every trainer: the construction with its parameter check, the flat float32 master / momentum / gradient
    buffers and their views, the launch layer over one image -- _conv, _prep, _pool, _chw, the cached gradient buffers and
    the in-place repack -- the weight gradients, the RPN forward, the gradient exchange and the optimizer.  _CanvasSteps
    overrides the launches for a canvas, so every step is written once.  The trunk supplies feat_ch, halvings,
    first_layer, early_exchange, feat_grad_tag and the _trunk / _pack_image hooks; the step _step_table and repack."""

    def _init_common(self, params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                     lead=(), optimizer=None):
        """Checks the trunk's options and every parameter the trainer reads (FrcnnError before anything is allocated), then
        lays out the flat buffers over the trunk's convolutions and the step's convolutions and parameters, and the
        trunk's constants and activations.  lead: the leading [N] of a canvas trainer's activations.  optimizer: the rule
        (optimizers.MomentumSGD / Adam / AdaGrad / RMSprop), None for MomentumSGD(lr, momentum)."""
        optimizer = optimizers.resolve(optimizer, lr, momentum)
        layers, consts = self._trunk_table(H, W, feat_stride)
        step_layers, step_params, frozen = self._step_table(len(anchors))
        layers += step_layers
        entries = _entries(layers, step_params)
        for name, shape in entries + consts + frozen:
            got = tuple(np.shape(params[name])) if name in params else None
            if got != shape:
                raise FrcnnError("%s: parameter %s must have shape %s (got %s)" % (type(self).__name__, name, shape, got))
        self._init_params(params, H, W, anchors, precision, optimizer, weight_decay, feat_stride, device, process_group,
                          layers, entries, lead)
        self.x_in = torch.zeros(tuple(lead) + (3, H, W), dtype=torch.float32, device=self.device)
        self._init_trunk(params, H, W, lead)

    def _init_params(self, params, H, W, anchors, precision, optimizer, weight_decay, feat_stride, device, process_group,
                     layers, entries, lead=()):
        """Hyper-parameters, the flat float32 master / optimizer-state / gradient buffers over `entries` ([(name, shape)], stored
        in the given order with NO padding: adjacent twin heads stay one matrix; fc6/W in the RoI pooling's (h, w, c)
        column order), the activation allocator and the exchange state."""
        if precision not in ops.PRECISIONS:
            raise FrcnnError("precision must be one of %s" % (ops.PRECISIONS,))
        self.x3 = precision == "bf16x3"
        self.precision, self.H, self.W = precision, H, W
        self.optimizer, self.weight_decay = optimizer, weight_decay
        self.feat_stride, self.pg = feat_stride, process_group
        dev = self.device = torch.device(device)
        self.anchors = torch.from_numpy(np.ascontiguousarray(anchors, dtype=np.float64)).to(dev)
        self.A = int(self.anchors.shape[0])
        # ---- trainable parameters in the reference's naming; one flat fp32 master / momentum / gradient buffer
        self.layers = layers
        sizes = [int(np.prod(s)) for _, s in entries]
        offs = [0] + [int(v) for v in np.cumsum(sizes)[:-1]]
        total = int(sum(sizes))
        self.w_flat = torch.zeros((total,), dtype=torch.float32, device=dev)
        # the rule's state ({"v"}, Adam {"m", "v"}, AdaGrad {"h"}, RMSprop {"ms"}) in w_flat's layout; v_flat is
        # MomentumSGD's velocity (None under another rule); opt_t counts the rule's updates (Adam's t)
        self.opt_state = {k: torch.zeros_like(self.w_flat) for k in optimizer.states}
        self.v_flat = self.opt_state["v"] if optimizer.rule == optimizers.MOMENTUM_SGD else None
        self.opt_t = 0
        self.hyper = torch.zeros((optimizers.HYPER_LEN,), dtype=torch.float32, device=dev)   # what the update reads
        self._capturing = False
        self.g_flat = torch.zeros_like(self.w_flat)
        self.index = {}
        for (n, s), o, sz in zip(entries, offs, sizes):
            self.index[n] = (o, sz, s)
            src = _fc6_to_hwc(n, np.ascontiguousarray(params[n], dtype=np.float32))
            self.w_flat[o:o + sz] = torch.from_numpy(np.ascontiguousarray(src).reshape(-1)).to(dev)
        x3 = self.x3

        def act(h, w, c):
            hi = torch.empty(tuple(lead) + (h, w, c), dtype=torch.bfloat16, device=dev)
            return ops.Act(hi, torch.empty_like(hi) if x3 else None)

        self._act = act
        self._slots = int(lead[0]) if lead else 1           # images per step
        # the data gradients' bias: as wide as the widest one, fc6's into the 7x7 RoI pool (feat_ch * 49 outputs)
        self.zero_bias = torch.zeros((max(32768, 49 * self.feat_ch),), dtype=torch.float32, device=dev)
        # gradient activations (NHWC) and transposed buffers, shared between layers of identical shape
        self._acts, self._tbufs = {}, {}
        self.packed = {}
        self.last_losses = None
        # ---- multi-GPU gradient exchange (train_rpn.py:169-174): "fp32" = one exact SUM of the fp32 bucket (the parity
        # mode: bucket == sum of the per-image gradients bit for bit); "bf16" = BASELINE config #5: the bucket is rounded
        # to bf16 for the all-reduce (half the bytes), masters / momentum stay fp32.  The exchange runs on its own stream
        # in two buckets when the trunk names an early_exchange layer: the layers from it on (VGG16: conv4_1 ... heads, 90 %
        # of the parameters) are reduced while the shallower ones still back-propagate; else in one after backward.
        self.grad_dtype = "fp32"
        self.g_bf16 = None
        self.comm_stream = None
        self._comm_done = None
        self._bucket_lo = None              # flat offset where the early (deep-layer) bucket starts
        self.n_updates = 0                  # optimizer steps taken (the drop-in model syncs its Link params when this moves)
        self._ev_bwd = self._ev_comm = None

    # ---------------------------------------------------------------- views
    def view(self, flat, name):
        o, sz, shape = self.index[name]
        return flat[o:o + sz].view(shape)

    def weights(self, name):
        return self.view(self.w_flat, name)

    def grads(self, name):
        return self.view(self.g_flat, name)

    # ---------------------------------------------------------------- launches over one image (_CanvasSteps: a canvas)
    def _conv(self, x, planes, bias, ksize, relu, at, **kw):
        """frcnn_conv2d.  at: where the rows live -- a trunk level (nothing to pass for one image; on a canvas
        _CanvasSteps._level resolves it), "rois": the head's forward, which computes the first prop.count rows, or
        "roi_grads": the head's data gradients."""
        if at == "rois":
            kw["m_valid"] = self.prop.count
        return ops.conv2d(x, planes[0], planes[1], bias, ksize, relu, **kw)

    def _prep(self, h, w, c, **kw):
        train_ops.grad_prepare(h, w, c, **kw)

    def _pool(self, y, out):
        ops.maxpool2x2_ceil(y, out=out)

    def _pack_input(self, x_chw):
        """The trunk's first launch: the image into the first layer's im2col planes x_col."""
        self.x_in.copy_(x_chw, non_blocking=True)
        self._pack_image(self.x_in, self.x_col)

    # the ResNet trunk's launches (resnet_train._ResNetTrunk); `at` as in _conv
    def _res_conv(self, x, planes, bias, ksize, relu, res, at, out):
        """frcnn_conv2d_res: y = act(conv(x) + bias + res)."""
        ops.conv2d_res(x, planes[0], planes[1], bias, ksize, relu, res, out=out)

    def _pool3(self, y, out, at):
        """The 3x3/2 cover_all max-pool of y (at: y's level)."""
        ops.maxpool3x3s2_ceil(y, out=out)

    def _subsample(self, x, out):
        ops.subsample2x(x, out=out)

    def _pool3_backward(self, g, y, p, out, tbuf):
        train_ops.maxpool3x3s2_backward(g, y, p, out=out, tbuf=tbuf)

    def _prep_stride2(self, h, w, c, g, y, out, tbuf):
        train_ops.grad_prepare_stride2(h, w, c, g, y=y, out=out, tbuf=tbuf)

    def _chw(self, act):
        """float32 (C,H,W) copy of an Act (debug)."""
        return act.to_chw_f32()

    def _gact(self, h, w, c, tag=0):
        """A gradient activation, shared between layers of identical shape and tag."""
        key = (h, w, c, tag)
        if key not in self._acts:
            self._acts[key] = self._act(h, w, c)
        return self._acts[key]

    def _tbuf(self, planes, c, h, w, tag=0):
        key = (planes, c, h, w, tag)
        if key not in self._tbufs:
            self._tbufs[key] = train_ops.TBuf(planes, c, h, w, self.device, self.x3, N=self._slots)
        return self._tbufs[key]

    # ---------------------------------------------------------------- weights: repacked in place from the fp32 masters
    def _repack(self, name, w, b, cout_pad, first=False, cin_pad=None):
        """packed[name] = (forward planes, padded bias, data-gradient planes or None for the first layer), overwriting the
        earlier tensors: a captured graph, and whoever else holds them, reads the new weights."""
        old = self.packed.get(name)
        if first:
            fwd, dg = self._pack_image_layer(w, out=old and old[0]), None
        else:
            fwd = ops.pack_conv_weights(w, cin_pad=cin_pad, precision=self.precision, out=old and old[0])
            dg = train_ops.pack_conv_weights_dgrad(w, cout_pad=cout_pad, x3=self.x3, out=old and old[2])
        self.packed[name] = (fwd, ops.pad_bias(b, cout_pad, out=old and old[1]), dg)

    # ---------------------------------------------------------------- forward
    def _rpn_forward(self, x, conv, heads, mid, ld, out):
        """An RPN on the feature map x: its 3x3 conv + ReLU into `mid`, its twin 1x1 heads into the fp32 [rows, ld] `out`.
        conv / heads: (planes, bias, ...) -- the trained layers' `packed` entries or the RCNN step's frozen ones."""
        self._conv(x, conv[0], conv[1], 3, True, self.halvings, out=mid)
        self._conv(mid, heads[0], heads[1], 1, False, self.halvings, out_act=False, ld_f32=ld, out_f32=out)

    # ---------------------------------------------------------------- weight gradients
    def _splits(self, groups, M, N, kb_total):
        # measured (tests/gpu_wgrad_tune.py): ~2 waves of 148 tiles, 4 when the M tile is half empty (64 output channels)
        tiles = groups * ((M + 127) // 128) * ((N + 127) // 128)
        target = (4 if M <= 64 else 2) * 148
        s = max(1, (target + tiles - 1) // tiles)
        return int(min(s, max(1, kb_total // 8)))

    def _wgrad(self, dyT, xT, M, N, groups, dw, m_out=None, scale=None):
        """dw (flat view) = sum_pixels dY (x) X over the padded pixel axis; dyT: TBuf 1 plane [M_parts, Kp]; xT: TBuf.
        scale: float64 [M] per-output-channel factor (a frozen BatchNorm's s), applied in the fixed-order reduction."""
        K = dyT.hi.shape[-1]                    # N*Kp: a canvas sums its N images in the one GEMM
        a_hi, a_lo = dyT.hi[0], (dyT.lo[0] if dyT.lo is not None else None)
        if groups == 9:
            b_hi, b_lo = xT.hi, xT.lo
        else:
            pl = 1 if xT.planes == 3 else 0
            b_hi, b_lo = xT.hi[pl], (xT.lo[pl] if xT.lo is not None else None)
        parts = train_ops.gemm_nt_splitk(a_hi, a_lo, b_hi, b_lo, groups=groups, row_stride=dyT.Wp,
                                         splits=self._splits(groups, M, N, K // 64))
        if scale is None:
            train_ops.wgrad_reduce(parts, m_out or M, N, dw)
        else:
            train_ops.wgrad_reduce_scaled(parts, m_out or M, N, scale, dw)

    def _first_layer_wgrad(self, dyT, h, w, co, dw, scale=None):
        """The first convolution's weight gradient into dw (OIHW [co][3][k][k]) from dyT and its im2col input x_col: the
        GEMM over the K_pad columns (scaled as _wgrad scales), then im2col column tap*3 + c -> OIHW [co][c][tap]."""
        k, _, _, K_pad = self.first_layer
        xT = self._tbuf(1, K_pad, h, w)
        self._prep(h, w, K_pad, g=self.x_col, tbuf=xT)
        dwc = torch.empty((co, K_pad), dtype=torch.float32, device=self.device)
        self._wgrad(dyT, xT, co, K_pad, 1, dwc, scale=scale)
        dw.copy_(dwc[:, :3 * k * k].reshape(co, k * k, 3).permute(0, 2, 1).reshape(co, 3, k, k))

    # ---------------------------------------------------------------- gradient exchange + optimizer
    def set_grad_exchange(self, grad_dtype="fp32", overlap=True):
        """grad_dtype "fp32" (exact) or "bf16" (config #5); overlap: reduce the deep-layer bucket during the rest of backward."""
        if grad_dtype not in ("fp32", "bf16"):
            raise FrcnnError("grad_dtype must be fp32 or bf16")
        self.grad_dtype = grad_dtype
        if grad_dtype == "bf16" and self.g_bf16 is None:
            self.g_bf16 = torch.zeros(self.g_flat.shape, dtype=torch.bfloat16, device=self.device)
        self._overlap = bool(overlap)

    def _multi(self):
        return shard.dist.is_available() and shard.dist.is_initialized() and shard.dist.get_world_size(self.pg) > 1

    def _exchange(self, lo, hi):
        """All-reduce(SUM) of g_flat[lo:hi] on the communication stream, after everything queued so far on the compute stream."""
        if self.comm_stream is None:
            self.comm_stream = torch.cuda.Stream(device=self.device)
        ev = torch.cuda.Event()
        ev.record()
        self.comm_stream.wait_event(ev)
        with torch.cuda.stream(self.comm_stream):
            if self.grad_dtype == "bf16":
                train_ops.cast_f32_bf16(self.g_flat[lo:hi], self.g_bf16[lo:hi])
                shard.allreduce_sum_(self.g_bf16[lo:hi], self.pg)
            else:
                shard.allreduce_sum_(self.g_flat[lo:hi], self.pg)

    def _early_exchange(self, layer_name):
        """Called from the trunk's backward right after `layer_name`'s gradients are enqueued: at the trunk's
        early_exchange layer, starts the exchange of the deep-layer bucket."""
        if not getattr(self, "_overlap", True) or not self._multi() or layer_name != self.early_exchange:
            return
        lo = self.index[layer_name + "/W"][0]
        if lo % 4 != 0:
            return
        self._bucket_lo = lo
        self._exchange(lo, self.g_flat.numel())

    # ---------------------------------------------------------------- the rule's hyper-parameters and state
    @property
    def lr(self):
        """The rule's learning rate: `optimizer.lr`, Adam's `optimizer.alpha`."""
        return getattr(self.optimizer, self.optimizer.lr_name)

    @lr.setter
    def lr(self, value):
        setattr(self.optimizer, self.optimizer.lr_name, value)

    @property
    def momentum(self):
        """MomentumSGD's momentum (AttributeError under another rule)."""
        if self.optimizer.rule != optimizers.MOMENTUM_SGD:
            raise AttributeError("%s has no momentum" % type(self.optimizer).__name__)
        return self.optimizer.momentum

    @momentum.setter
    def momentum(self, value):
        if self.optimizer.rule != optimizers.MOMENTUM_SGD:
            raise AttributeError("%s has no momentum" % type(self.optimizer).__name__)
        self.optimizer.momentum = value

    def _write_hyper(self):
        """The next update's hyper-parameters (the current optimizer values, weight_decay and t + 1) into the device array
        the update reads: one stream-ordered host-to-device copy from pinned memory, which the caching host allocator keeps
        until the copy has run, so nothing waits.  Raises FrcnnError for a bad value before anything is queued."""
        self.optimizer.check()
        vals = torch.from_numpy(self.optimizer.hyper(self.weight_decay, self.opt_t + 1))
        self.hyper.copy_(vals.pin_memory() if self.hyper.is_cuda else vals, non_blocking=True)
        self.opt_t += 1

    def _optimizer_update(self, g):
        s = [self.opt_state[k] for k in self.optimizer.states]
        train_ops.optimizer_update(self.optimizer.rule, self.w_flat, s[0], s[1] if len(s) > 1 else None, g, self.hyper)

    def optimizer_state(self, to_host=True):
        """The rule's state under the reference's parameter names: {"rule": name, "t": updates taken, state name: {param:
        array}} with fp32 arrays in the reference's layouts (fc6/W in (c, h, w) column order, as export_params);
        to_host=False: device tensors (copies) instead of NumPy arrays."""
        out = {"rule": type(self.optimizer).__name__, "t": self.opt_t}
        for k, buf in self.opt_state.items():
            out[k] = self._host_arrays(buf) if to_host else {n: self._ref_layout(n, self.view(buf, n)).clone() for n in self.index}
        return out

    def load_optimizer_state(self, state):
        """Loads what optimizer_state returned (NumPy arrays or tensors) for the same rule and parameters."""
        who = type(self).__name__
        if state.get("rule") != type(self.optimizer).__name__:
            raise FrcnnError("%s.load_optimizer_state: the state is %r's, the trainer runs %s"
                             % (who, state.get("rule"), type(self.optimizer).__name__))
        for k in self.opt_state:
            if k not in state or set(state[k]) != set(self.index):
                raise FrcnnError("%s.load_optimizer_state: state %r must hold every trained parameter" % (who, k))
            for n, a in state[k].items():
                if tuple(a.shape) != self.index[n][2]:
                    raise FrcnnError("%s.load_optimizer_state: %s/%s has shape %s, needs %s"
                                     % (who, k, n, tuple(a.shape), self.index[n][2]))
        for k, buf in self.opt_state.items():
            for n, a in state[k].items():
                t = torch.as_tensor(a, dtype=torch.float32)
                self.view(buf, n).copy_(t.reshape(4096, -1, 49).transpose(1, 2).reshape(4096, -1) if n == "fc6/W" else t)
        self.opt_t = int(state["t"])

    def update(self):
        """[all-reduce SUM over ranks, like ParallelUpdater's addgrads] + WeightDecay + the optimizer's rule, then repack.
        The hyper-parameters are written before the update is queued, except inside a capture (_CanvasSteps._step writes
        them before each replay)."""
        if self._multi():
            hi = self._bucket_lo if self._bucket_lo is not None else self.g_flat.numel()
            self._ev_bwd = torch.cuda.Event(enable_timing=True)
            self._ev_bwd.record()                                  # backward fully enqueued on the compute stream
            self._exchange(0, hi)
            self._ev_comm = torch.cuda.Event(enable_timing=True)
            self._ev_comm.record(self.comm_stream)
            torch.cuda.current_stream().wait_event(self._ev_comm)
            self._bucket_lo = None
        if not self._capturing:
            self._write_hyper()
        self._optimizer_update(self.g_bf16 if self.grad_dtype == "bf16" and self._multi() else self.g_flat)
        self.repack()
        self.n_updates += 1

    def last_exposed_exchange_ms(self):
        """Time between "backward done" on the compute stream and "exchange done" on the communication stream for the last
        step (what the optimizer had to wait for); call after a synchronize.  0 if the exchange finished first."""
        if self._ev_bwd is None or self._ev_comm is None:
            return 0.0
        return max(0.0, self._ev_bwd.elapsed_time(self._ev_comm))

    def _ref_layout(self, name, a):
        """A parameter-shaped view of a flat buffer in the reference's layout: fc6/W's (h, w, c) columns back to (c, h, w)."""
        return a.reshape(4096, 49, -1).transpose(1, 2).reshape(4096, -1) if name == "fc6/W" else a

    def _host_arrays(self, flat):
        return {n: self._ref_layout(n, self.view(flat, n)).detach().cpu().numpy().copy() for n in self.index}

    def export_params(self):
        """Trainable parameters as numpy arrays under the reference's names and layouts (fc6/W in (c, h, w) column order):
        checkpoint / write-back into the Links."""
        return self._host_arrays(self.w_flat)


class _Vgg16Trunk(object):
    """The VGG16 trunk: 13 3x3 convolutions, the first on the image's 3x3 im2col planes, with every output kept (pools
    un-fused: backward needs the un-pooled maps); the feature map is conv5_3's output at 1/16."""
    feat_ch = 512                   # channels of the feature map the RPN and the RoI pooling read (conv5_3)
    halvings = 4                    # the feature map's canvas level: after four 2x2 pools
    first_layer = (3, 1, 1, 32)     # ksize, stride, pad, K_pad of the first layer's im2col input
    early_exchange = "trunk/conv4_1"    # the deep bucket of the gradient exchange: conv4_1 on, 90 % of the parameters
    feat_grad_tag = 1               # the _gact tag of the trunk's data gradients, which the RPN conv's data gradient shares

    def _trunk_table(self, H, W, feat_stride):
        """The trunk's convolutions in flat-buffer order and the constants it reads besides them (none)."""
        return [dict(name="trunk/" + n, cin=ci, cout=co, k=3) for n, ci, co in TRUNK], []

    def _init_trunk(self, params, H, W, lead):
        """Geometry + activations: every conv output, and the pooled maps where the graph pools; `lead`: the leading [N]
        of a canvas trainer's activations, whose extents at a layer are ceil(extent / 2^halvings)."""
        act = self._act
        self.x_col = act(H, W, 32)
        h, w, halvings = H, W, 0
        for L in self.layers[:13]:
            L["H"], L["W"], L["halvings"] = h, w, halvings
            L["y"] = act(h, w, L["cout"])
            short = L["name"].split("/")[1]
            L["pool"] = short in POOL_AFTER
            if L["pool"]:
                h, w, halvings = (h + 1) // 2, (w + 1) // 2, halvings + 1
                L["p"] = act(h, w, L["cout"])
        self.fh, self.fw = h, w

    def _pack_image(self, x, out):
        """The first layer's im2col planes of one image."""
        ops.pack_image_im2col(x, out=out)

    def _pack_image_layer(self, w, out=None):
        """The first convolution's planes, in the K order of the trunk's im2col input."""
        return ops.pack_conv_weights_im2col(w, precision=self.precision, out=out)

    def _repack_trunk(self):
        for i, L in enumerate(self.layers[:13]):
            name = L["name"]
            self._repack(name, self.weights(name + "/W"), self.weights(name + "/b"), L["cout"], first=i == 0, cin_pad=L["cin"])

    def _forward_trunk(self, x_chw=None):
        """The 13 VGG16 convolutions with every output kept (pools un-fused: backward needs the un-pooled maps)."""
        self._pack_input(x_chw)
        x = self.x_col
        for i, L in enumerate(self.layers[:13]):
            fwd, b, _ = self.packed[L["name"]]
            self._conv(x, fwd, b, 1 if i == 0 else 3, True, L["halvings"], out=L["y"])
            x = L["y"]
            if L["pool"]:
                self._pool(L["y"], out=L["p"])
                x = L["p"]
        self.feat = x
        return x

    def _backward_trunk(self, g, debug=None):
        """Backward through the 13 convolutions, last first, from g: the gradient (ops.Act) w.r.t. the feature map.  Per
        layer: ReLU / pool backward + re-layout, weight + bias gradient, data gradient for the next one.  On a canvas the
        weight gradients run over K = N*Kp, the sum over the slots.  debug: per layer name, "g_in", "dy" and (but for
        conv1_1) "g_out", as the step's backward describes them."""
        for L in self.layers[12::-1]:
            h, w, co, ci = L["H"], L["W"], L["cout"], L["cin"]
            first = L is self.layers[0]
            dy = self._gact(h, w, co)
            dyT = self._tbuf(1, co, h, w)
            self._prep(h, w, co, g=g, y=L["y"], p=L.get("p") if L["pool"] else None, out=dy, tbuf=dyT)
            if debug is not None:
                debug[L["name"]] = dict(g_in=self._chw(g), dy=self._chw(dy))
            if first:
                self._first_layer_wgrad(dyT, h, w, co, self.grads(L["name"] + "/W"))
            else:
                xT = self._tbuf(3, ci, h, w)
                self._prep(h, w, ci, g=self._input_of(L), tbuf=xT)
                self._wgrad(dyT, xT, co, ci, 9, self.grads(L["name"] + "/W"))
            train_ops.bias_grad(dyT, co, self.grads(L["name"] + "/b"))
            self._early_exchange(L["name"])
            if not first:
                g = self._gact(h, w, ci, tag=self.feat_grad_tag)
                self._conv(dy, self.packed[L["name"]][2], self.zero_bias, 3, False, L["halvings"], out=g)
                if debug is not None:
                    debug[L["name"]]["g_out"] = self._chw(g)

    def _input_of(self, L):
        i = self.layers.index(L)
        if i == 0:
            return self.x_col
        if i == 13:
            return self.feat
        prev = self.layers[i - 1]
        return prev["p"] if prev["pool"] else prev["y"]


class _RpnStep(_ConvTrainer):
    """The RPN step over any trunk: the RPN 3x3 conv and its twin heads, AnchorTargetLayer, rpn_loss and the backward
    through the heads and the RPN conv into the trunk's.

    The names the RCNN step also uses for its own head -- the twin heads' `packed` key, head_ld, n_heads, head_out,
    head_grad, delta and targets -- live on `_rpn`: the trainer itself, or in _JointStep, which holds both steps, an
    _RpnNames beside the RCNN step's."""
    heads_key = "heads"         # the twin heads' entry in `packed`

    @property
    def _rpn(self):
        return self

    def _init_rpn(self, params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                  loss_lambda, delta, subsample, seed, optimizer=None):
        self._init_common(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                          optimizer=optimizer)
        self._init_rpn_head(loss_lambda, delta, subsample, seed)
        self._rpn.targets = train_ops.AnchorTargets(self.A, self.fh, self.fw, self.device)
        self.repack()

    def _step_table(self, A):
        """The step's convolutions and parameters in flat-buffer order, and the parameters it reads but does not train.
        The twin heads are stored adjacently so that (W_cls | W_bbox) is ONE [6A, 512] matrix: cls W, bbox W, cls b, bbox b."""
        heads = [("RPN/rpn_cls_score", 2 * A), ("RPN/rpn_bbox_pred", 4 * A)]
        return ([dict(name="RPN/rpn_conv_3x3", cin=self.feat_ch, cout=512, k=3)],
                [(n + "/W", (co, 512, 1, 1)) for n, co in heads] + [(n + "/b", (co,)) for n, co in heads], [])

    def _init_rpn_head(self, loss_lambda, delta, subsample, seed):
        """The RPN step's loss settings, its 3x3 conv (the last layer) at the feature map and the twin heads' output."""
        r = self._rpn
        self.loss_lambda, self.subsample, self.seed = loss_lambda, subsample, seed
        r.delta = delta
        r.n_heads = 6 * self.A
        r.head_ld = ops.round_up(r.n_heads, 32)
        R = self.rpn_layer = self.layers[-1]
        R["H"], R["W"], R["pool"], R["halvings"] = self.fh, self.fw, False, self.halvings
        R["y"] = self._act(self.fh, self.fw, 512)
        r.head_out = torch.empty((self._slots * self.fh * self.fw, r.head_ld), dtype=torch.float32, device=self.device)

    def _rpn_heads_w(self, flat):
        o, _, _ = self.index["RPN/rpn_cls_score/W"]
        return flat[o:o + self._rpn.n_heads * 512].view(self._rpn.n_heads, 512)

    def _rpn_heads_b(self, flat):
        o, _, _ = self.index["RPN/rpn_cls_score/b"]
        return flat[o:o + self._rpn.n_heads]

    def repack(self):
        self._repack_trunk()
        self._repack_rpn()

    def _repack_rpn(self):
        R, r = self.rpn_layer, self._rpn
        self._repack(R["name"], self.weights(R["name"] + "/W"), self.weights(R["name"] + "/b"), 512, cin_pad=R["cin"])
        self._repack(r.heads_key, self._rpn_heads_w(self.w_flat), self._rpn_heads_b(self.w_flat), r.head_ld)

    # ---------------------------------------------------------------- forward
    def forward(self, x_chw, gt_boxes, im_info=None, disable_pos=None):
        """x_chw (3,H,W) float32 CUDA; gt_boxes [G,5] float32 CUDA.  Returns losses float32[4] (device):
        rpn_loss_cls, rpn_loss_bbox, rpn_cls_accuracy, rpn_loss.  (The reference also runs the ProposalLayer here,
        region_proposal_network.py:122-124; its output does not enter the RPN loss and is skipped.)"""
        im_h, im_w = (self.H, self.W) if im_info is None else (int(im_info[0]), int(im_info[1]))
        self._rpn_trained_forward(self._forward_trunk(x_chw))
        self.last_losses = self._rpn_losses(gt_boxes, im_h, im_w, disable_pos)
        return self.last_losses

    def _rpn_trained_forward(self, feat):
        """The trained RPN (its `packed` planes) on the feature map: rpn_layer's y and the twin heads' _rpn.head_out."""
        R, r = self.rpn_layer, self._rpn
        self._rpn_forward(feat, self.packed[R["name"]], self.packed[r.heads_key], R["y"], r.head_ld, r.head_out)

    def _rpn_losses(self, gt_boxes, im_h, im_w, disable_pos):
        """AnchorTargetLayer and rpn_loss on _rpn.head_out; sets _rpn.head_grad.  Returns losses float32[4] (device)."""
        r = self._rpn
        if disable_pos is None and self.subsample == "numpy":
            disable_pos = self._numpy_subsample(gt_boxes, im_h, im_w)
        if disable_pos is not None:
            mode, kw = train_ops.SUBSAMPLE_LIST, dict(disable_pos=disable_pos)
        elif self.subsample == "device":
            mode, kw = train_ops.SUBSAMPLE_DEVICE, dict(seed=self.seed)
            self.seed += 1
        else:
            mode, kw = train_ops.SUBSAMPLE_NONE, {}
        train_ops.anchor_targets(self.anchors, self.A, self.fh, self.fw, self.feat_stride, gt_boxes, im_h, im_w, mode=mode,
                                 work=r.targets, **kw)
        losses, r.head_grad, _ = train_ops.rpn_loss(r.head_out, None, self.anchors, self.A, self.fh, self.fw,
                                                    self.feat_stride, im_h, im_w, r.targets, delta=r.delta,
                                                    loss_lambda=self.loss_lambda, layout="nhwc", ld=r.head_ld)
        return losses

    def _numpy_subsample(self, gt_boxes, im_h, im_w):
        """The reference's own subsampling (anchor_target_layer.py:148-168): labels before subsampling come back to the host
        and np.random.choice draws from NumPy's global RNG in the reference's order (a seeded run reproduces the reference's
        labels bit for bit); returns the positions to disable in the inside-compact numbering (int32 CUDA tensor)."""
        w = train_ops.anchor_targets(self.anchors, self.A, self.fh, self.fw, self.feat_stride, gt_boxes, im_h, im_w,
                                     mode=train_ops.SUBSAMPLE_NONE, work=self._rpn.targets)
        n_inside = int(w.counts[0].item())
        labels = w.labels_full[w.inds_inside[:n_inside].long()].cpu().numpy()
        num_fg = int(train_ops.RPN_FG_FRACTION * train_ops.RPN_BATCHSIZE)
        disable = [np.zeros((0,), np.int64)]
        fg_inds = np.where(labels == 1)[0]
        if len(fg_inds) > num_fg:
            d = np.random.choice(fg_inds, size=int(len(fg_inds) - num_fg), replace=False)
            labels[d] = -1
            disable.append(d)
        num_bg = train_ops.RPN_BATCHSIZE - np.sum(labels == 1)
        bg_inds = np.where(labels == 0)[0]
        if len(bg_inds) > num_bg:
            disable.append(np.random.choice(bg_inds, size=int(len(bg_inds) - num_bg), replace=False))
        return torch.from_numpy(np.concatenate(disable).astype(np.int32)).to(self.device)

    # ---------------------------------------------------------------- backward
    def backward(self, debug=None):
        """Fills g_flat with d(rpn_loss)/d(parameter) for every trainable parameter (on a canvas: the sum over the slots).
        debug: a dict that receives, per layer name, float32 (C,H,W) copies ([N,C,H,W] on a canvas) of the incoming
        gradient ("g_in"), the masked / routed gradient ("dy") and the data gradient the layer passes on ("g_out") -- the
        buffers themselves are reused from layer to layer.  The trunk's entries are those of its _backward_trunk."""
        self._backward_trunk(self._backward_rpn(debug), debug)

    def _backward_rpn(self, debug=None, res=None, tag=None):
        """The twin heads' and the RPN 3x3 conv's (feat_ch -> 512, its own bias) gradients; returns the RPN conv's data
        gradient, the gradient of the feature map, in the _gact of `tag` (default the trunk's feat_grad_tag).  res: a
        gradient of the feature map from elsewhere (ops.Act, another buffer), added in the data gradient's epilogue
        (frcnn_conv2d_res)."""
        g = self._backward_heads(debug)
        R, fh, fw, C = self.rpn_layer, self.fh, self.fw, self.feat_ch
        dy = self._gact(fh, fw, 512)
        dyT = self._tbuf(1, 512, fh, fw)
        self._prep(fh, fw, 512, g=g, y=R["y"], out=dy, tbuf=dyT)
        if debug is not None:
            debug[R["name"]] = dict(g_in=self._chw(g), dy=self._chw(dy))
        xT = self._tbuf(3, C, fh, fw)
        self._prep(fh, fw, C, g=self.feat, tbuf=xT)
        self._wgrad(dyT, xT, 512, C, 9, self.grads(R["name"] + "/W"))
        train_ops.bias_grad(dyT, 512, self.grads(R["name"] + "/b"))
        g = self._gact(fh, fw, C, tag=self.feat_grad_tag if tag is None else tag)
        if res is None:
            self._conv(dy, self.packed[R["name"]][2], self.zero_bias, 3, False, self.halvings, out=g)
        else:
            self._res_conv(dy, self.packed[R["name"]][2], self.zero_bias, 3, False, res, self.halvings, g)
        if debug is not None:
            debug[R["name"]]["g_out"] = self._chw(g)
        return g

    def _backward_heads(self, debug=None):
        """The twin 1x1 heads' weight / bias gradients; returns the gradient w.r.t. the RPN 3x3 conv's post-ReLU output.
        debug: the entry under _rpn.heads_key."""
        r = self._rpn
        fh, fw, ld = self.fh, self.fw, r.head_ld
        R = self.rpn_layer
        # ---- twin 1x1 heads: dY = head_grad [fh*fw, ld] fp32 (columns >= 6A are zero)
        dyh = self._gact(fh, fw, ld)
        dyhT = self._tbuf(1, ld, fh, fw)
        self._prep(fh, fw, ld, g_f32=r.head_grad, out=dyh, tbuf=dyhT)
        midT = self._tbuf(3, 512, fh, fw)
        self._prep(fh, fw, 512, g=R["y"], tbuf=midT)
        self._wgrad(dyhT, midT, ld, 512, 1, self._rpn_heads_w(self.g_flat), m_out=r.n_heads)
        train_ops.bias_grad(dyhT, r.n_heads, self._rpn_heads_b(self.g_flat))
        g = self._gact(fh, fw, 512, tag=1)
        self._conv(dyh, self.packed[r.heads_key][2], self.zero_bias, 1, False, self.halvings, out=g)
        if debug is not None:
            debug[r.heads_key] = dict(dy=self._chw(dyh), g_out=self._chw(g))
        return g

    def step(self, x_chw, gt_boxes, im_info=None, disable_pos=None):
        losses = self.forward(x_chw, gt_boxes, im_info, disable_pos)
        self.backward()
        self.update()
        return losses


class _RcnnStep(_ConvTrainer):
    """The RCNN step over any trunk: the frozen test-mode RPN, ProposalLayer, ProposalTargetLayer, RoI pooling, fc6 / fc7
    with dropout, cls_score | bbox_pred, the losses and the backward through the head and the RoI pooling into the trunk's.
    fc6/W is kept in the (h, w, c) input order the RoI-pool kernel emits (`export_params` converts back)."""

    def _init_rcnn(self, params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                   num_classes, delta, post_n, pre_n, nms_thresh, min_size, sample, seed, dropout, optimizer=None):
        self.num_classes = num_classes
        self._init_common(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                          optimizer=optimizer)
        self._frozen_rpn(params)
        self._init_rcnn_head(delta, post_n, pre_n, nms_thresh, min_size)
        self._init_rcnn_draws(sample, seed, dropout)
        self.repack()

    def _init_rcnn_draws(self, sample, seed, dropout):
        """One image's sampling and dropout settings, the masks' generator and the proposal workspace."""
        self.sample, self.dropout = sample, dropout
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(seed)
        self.prop = ops.ProposalWorkspace(self.A, self.fh, self.fw, self.pre_n, self.post_n, self.device)
        self.roi_ws = None

    def _step_table(self, A):
        """The step's convolutions (none) and parameters in flat-buffer order (cls_score | bbox_pred adjacent: one
        [5*nc, 4096] matrix; fc6 reads the 7x7 RoI pool of the feature map), and the frozen RPN: the RPN step's parameters."""
        heads = [("cls_score", self.num_classes), ("bbox_pred", 4 * self.num_classes)]
        fc = [("fc6/W", (4096, self.feat_ch * 49)), ("fc6/b", (4096,)), ("fc7/W", (4096, 4096)), ("fc7/b", (4096,))]
        frozen_rpn = _entries(*_RpnStep._step_table(self, A)[:2])
        return [], fc + [(n + "/W", (co, 4096)) for n, co in heads] + [(n + "/b", (co,)) for n, co in heads], frozen_rpn

    def _init_rcnn_head(self, delta, post_n, pre_n, nms_thresh, min_size):
        """The head's settings and activations."""
        self.delta = delta
        self.post_n, self.pre_n, self.nms_thresh, self.min_size = post_n, pre_n, nms_thresh, min_size
        self.n_heads = 5 * self.num_classes
        self.head_ld = ops.round_up(self.n_heads, 32)
        dev, rows, C = self.device, self._slots * self.fh * self.fw, self.feat_ch
        self.pool5 = self._act(1, post_n, 49 * C)
        self.fc6 = self._act(1, post_n, 4096)
        self.fc7 = self._act(1, post_n, 4096)
        self.head_out = torch.empty((self._slots * post_n, self.head_ld), dtype=torch.float32, device=dev)
        self.dfeat = torch.empty((rows, C), dtype=torch.float32, device=dev)

    def _frozen_rpn(self, params):
        """The RPN's 3x3 and twin-head weights as (planes, bias), packed once (forward only: the RCNN step gives them no
        gradient), and their outputs."""
        T = lambda k: torch.from_numpy(np.ascontiguousarray(params[k], dtype=np.float32)).to(self.device)     # noqa: E731
        self.rpn3 = (ops.pack_conv_weights(T("RPN/rpn_conv_3x3/W"), cin_pad=self.feat_ch, precision=self.precision),
                     ops.pad_bias(T("RPN/rpn_conv_3x3/b"), 512))
        wh = torch.cat([T("RPN/rpn_cls_score/W"), T("RPN/rpn_bbox_pred/W")], dim=0)
        bh = torch.cat([T("RPN/rpn_cls_score/b"), T("RPN/rpn_bbox_pred/b")], dim=0)
        self.rpn_ld = ops.round_up(6 * self.A, 32)
        self.rpn_heads = (ops.pack_conv_weights(wh, precision=self.precision), ops.pad_bias(bh, self.rpn_ld))
        self.rpn_mid = self._act(self.fh, self.fw, 512)
        self.rpn_out = torch.empty((self._slots * self.fh * self.fw, self.rpn_ld), dtype=torch.float32, device=self.device)

    # ---------------------------------------------------------------- parameters
    def _heads_w(self, flat):
        o, _, _ = self.index["cls_score/W"]
        return flat[o:o + self.n_heads * 4096].view(self.n_heads, 4096)

    def _heads_b(self, flat):
        o, _, _ = self.index["cls_score/b"]
        return flat[o:o + self.n_heads]

    def repack(self):
        self._repack_trunk()
        self._repack_rcnn()

    def _repack_rcnn(self):
        for n in ("fc6", "fc7"):
            self._repack(n, self.weights(n + "/W"), self.weights(n + "/b"), 4096)
        self._repack("heads", self._heads_w(self.w_flat), self._heads_b(self.w_flat), self.head_ld)

    # ---------------------------------------------------------------- ProposalTargetLayer sampling (host, like the reference)
    def _sample(self, max_ov, R):
        mo = max_ov[:R].cpu().numpy()
        n_fg_cap = int(FG_FRACTION * ROIS_PER_IMAGE)
        fg = np.where(mo >= FG_THRESH)[0]                                                    # :99
        n_fg = min(n_fg_cap, fg.size)
        if fg.size > 0:
            fg = np.random.choice(fg, size=n_fg, replace=False)                              # :105-110
        bg = np.where((mo < BG_THRESH_HI) & (mo >= BG_THRESH_LO))[0]                         # :113-114
        n_bg = min(ROIS_PER_IMAGE - n_fg, bg.size)
        if bg.size > 0:
            bg = np.random.choice(bg, size=n_bg, replace=False)                              # :119-126
        return np.concatenate([fg, bg]).astype(np.int32)

    # ---------------------------------------------------------------- forward
    def forward(self, x_chw, gt_boxes, im_info=None, keep_inds=None, masks=None):
        """Returns losses float32[4] (device): loss_cls, loss_bbox, cls_accuracy, loss_rcnn."""
        im_h, im_w = (self.H, self.W) if im_info is None else (int(im_info[0]), int(im_info[1]))
        feat = self._forward_trunk(x_chw)
        self._rpn_forward(feat, self.rpn3, self.rpn_heads, self.rpn_mid, self.rpn_ld, self.rpn_out)
        self.last_losses = self._rcnn_losses(feat, self.rpn_out, self.rpn_ld, gt_boxes, im_h, im_w, keep_inds, masks)
        return self.last_losses

    def _rcnn_losses(self, feat, rpn_out, rpn_ld, gt_boxes, im_h, im_w, keep_inds, masks):
        """ProposalLayer on an RPN's output (fp32 [fh*fw, rpn_ld]: logits, then deltas), ProposalTargetLayer, RoI pooling,
        the head and its losses; sets head_grad.  Returns losses float32[4] (device)."""
        ops.proposals(rpn_out, None, self.anchors, self.A, self.fh, self.fw, self.feat_stride, im_h, im_w, self.min_size,
                      self.pre_n, self.post_n, self.nms_thresh, layout="nhwc", ld=rpn_ld, cls_is_logits=True, work=self.prop)
        rois, count = self.prop.rois, self.prop.count
        self.max_ov, self.argmax = train_ops.roi_overlaps(rois, count, gt_boxes)
        if keep_inds is None:
            R = int(count.item())                    # the reference sizes its arrays from len(proposals) too
            keep_inds = torch.from_numpy(self._sample(self.max_ov, R)).to(self.device)
        self.keep = keep_inds.to(device=self.device, dtype=torch.int32).contiguous()
        if self.keep.numel() < 1:
            raise FrcnnError("ProposalTargetLayer kept no RoI (no proposal overlaps a ground-truth box by >= 0.1)")
        self.use_gt, self.ext, self.labels = train_ops.roi_targets(rois, gt_boxes, self.argmax, self.keep, self.num_classes)
        ops.roi_pool(feat, rois, count, 7, 7, 1.0 / self.feat_stride, out=self.pool5)
        if masks is None and self.dropout:
            masks = [(torch.rand((self.post_n, 4096), device=self.device, generator=self.gen) >= 0.5).to(torch.uint8) for _ in range(2)]
        self.masks = masks
        self._head_forward()
        losses, self.head_grad = train_ops.rcnn_loss(self.head_out, self.keep, self.labels, self.ext, self.num_classes, self.delta)
        return losses

    def _head_forward(self):
        """fc6 -> fc7 -> cls_score | bbox_pred over the pooled RoIs into head_out, with `masks` dropout after fc6 and fc7."""
        fwd, b, _ = self.packed["fc6"]
        self._conv(self.pool5, fwd, b, 1, True, "rois", out=self.fc6)
        if self.masks is not None:
            train_ops.dropout_(self.fc6, self.masks[0])                                      # F.dropout(train=rcnn_train), :127
        fwd, b, _ = self.packed["fc7"]
        self._conv(self.fc6, fwd, b, 1, True, "rois", out=self.fc7)
        if self.masks is not None:
            train_ops.dropout_(self.fc7, self.masks[1])                                      # :128
        fwd, b, _ = self.packed["heads"]
        self._conv(self.fc7, fwd, b, 1, False, "rois", out_act=False, ld_f32=self.head_ld, out_f32=self.head_out)

    # ---------------------------------------------------------------- backward
    def _fc_wgrad(self, dyT, xT, M, N, dw, m_out=None):
        """dW [M][N] = dY^T X over the (padded) RoI axis; written straight into the gradient view when the shapes allow."""
        a_hi, a_lo = dyT.hi[0], (dyT.lo[0] if dyT.lo is not None else None)
        b_hi, b_lo = xT.hi[0], (xT.lo[0] if xT.lo is not None else None)
        if m_out is None and N % 32 == 0:
            train_ops.gemm_nt_splitk(a_hi, a_lo, b_hi, b_lo, groups=1, splits=1, out=dw.reshape(-1))
        else:
            parts = train_ops.gemm_nt_splitk(a_hi, a_lo, b_hi, b_lo, groups=1, splits=1)
            train_ops.wgrad_reduce(parts, m_out or M, N, dw)

    def backward(self, debug=None):
        """Fills g_flat with d(loss_rcnn)/d(parameter) for every trainable parameter.  debug: as RpnTrainer.backward, plus
        "roi": the gradient of the pooled RoIs ("dpool5") and of the feature map (fp32 [fh*fw, feat_ch], "dfeat")."""
        self._backward_trunk(self._backward_rcnn(debug), debug)

    def _backward_rcnn(self, debug=None):
        """The head's, fc7's and fc6's gradients and the RoI pooling's backward; returns the gradient of the feature map
        (dfeat split into the gradient activation of tag 3)."""
        R_cap, ld, C = self.post_n, self.head_ld, self.feat_ch
        twice = self.masks is not None               # ratio-0.5 dropout: dz = 2 * g * (y > 0), y = the post-dropout activation
        # ---- cls_score | bbox_pred: dY = head_grad [R_cap, ld] fp32 (zero rows for RoIs that were not kept)
        dyh = self._gact(1, R_cap, ld)
        dyhT = self._tbuf(1, ld, 1, R_cap)
        self._prep(1, R_cap, ld, g_f32=self.head_grad, out=dyh, tbuf=dyhT)
        fc7T = self._tbuf(1, 4096, 1, R_cap)
        self._prep(1, R_cap, 4096, g=self.fc7, tbuf=fc7T)
        self._fc_wgrad(dyhT, fc7T, ld, 4096, self._heads_w(self.g_flat), m_out=self.n_heads)
        train_ops.bias_grad(dyhT, self.n_heads, self._heads_b(self.g_flat))
        g = self._gact(1, R_cap, 4096, tag=1)
        self._conv(dyh, self.packed["heads"][2], self.zero_bias, 1, False, "roi_grads", out=g)
        if debug is not None:
            debug["heads"] = dict(dy=self._chw(dyh), g_out=self._chw(g))
        # ---- fc7
        dy7 = self._gact(1, R_cap, 4096)
        dy7T = self._tbuf(1, 4096, 1, R_cap, tag=1)
        self._prep(1, R_cap, 4096, g=g, y=self.fc7, out=dy7, tbuf=dy7T, times2=twice)
        if debug is not None:
            debug["fc7"] = dict(g_in=self._chw(g), dy=self._chw(dy7))
        fc6T = self._tbuf(1, 4096, 1, R_cap)          # the buffer of fc7T: the heads' weight gradient has consumed it
        self._prep(1, R_cap, 4096, g=self.fc6, tbuf=fc6T)
        self._fc_wgrad(dy7T, fc6T, 4096, 4096, self.grads("fc7/W"))
        train_ops.bias_grad(dy7T, 4096, self.grads("fc7/b"))
        g6 = self._gact(1, R_cap, 4096, tag=2)
        self._conv(dy7, self.packed["fc7"][2], self.zero_bias, 1, False, "roi_grads", out=g6)
        # ---- fc6
        dy6 = self._gact(1, R_cap, 4096)
        self._prep(1, R_cap, 4096, g=g6, y=self.fc6, out=dy6, tbuf=dy7T, times2=twice)       # dy7T's buffer now holds dy6^T
        if debug is not None:
            debug["fc6"] = dict(g_in=self._chw(g6), dy=self._chw(dy6))
        p5T = self._tbuf(1, 49 * C, 1, R_cap)
        self._prep(1, R_cap, 49 * C, g=self.pool5, tbuf=p5T)
        self._fc_wgrad(dy7T, p5T, 4096, 49 * C, self.grads("fc6/W"))
        train_ops.bias_grad(dy7T, 4096, self.grads("fc6/b"))
        gp = self._gact(1, R_cap, 49 * C, tag=1)
        self._conv(dy6, self.packed["fc6"][2], self.zero_bias, 1, False, "roi_grads", out=gp)
        # ---- RoI pooling backward -> gradient of the feature map, then the trunk
        self._roi_pool_backward(gp)
        gfeat = self._gact(self.fh, self.fw, C, tag=3)
        self._prep(self.fh, self.fw, C, g_f32=self.dfeat, out=gfeat)
        if debug is not None:
            debug["roi"] = dict(dpool5=self._chw(gp), dfeat=self.dfeat.clone())
        return gfeat

    def _roi_pool_backward(self, g):
        """dfeat = the RoI pooling's backward of g (the gradient of pool5)."""
        if self.roi_ws is None:
            self.roi_ws = torch.empty((ops._lib.load().frcnn_roi_pool_backward_workspace_bytes(self.fh, self.fw, self.feat_ch),),
                                      dtype=torch.uint8, device=self.device)
        train_ops.roi_pool_backward(self.feat, self.prop.rois, self.prop.count, g, 7, 7, 1.0 / self.feat_stride, out=self.dfeat,
                                    ws=self.roi_ws)

    def step(self, x_chw, gt_boxes, im_info=None, keep_inds=None, masks=None):
        losses = self.forward(x_chw, gt_boxes, im_info, keep_inds, masks)
        self.backward()
        self.update()
        return losses


class _RpnNames(object):
    """The RPN step's own head in _JointStep, where the trainer's head_ld, n_heads, head_out, head_grad, delta and
    packed["heads"] are the RCNN step's: the twin heads' `packed` key, width, output and gradient, rpn_loss's delta and the
    anchor targets."""
    heads_key = "RPN/heads"


JOIN_TAG = 4        # the _gact tag of the joined feature-map gradient: no trunk's backward uses it, so it is never the
                    # split dfeat (tag 3) it adds


class _JointStep(_RpnStep, _RcnnStep):
    """Approximate joint training (py-faster-rcnn's end2end recipe) over any trunk: one trunk forward, the trained RPN run
    once, AnchorTargetLayer and rpn_loss on its output, ProposalLayer on the same logits (the proposals are constants),
    ProposalTargetLayer, RoI pooling, fc6 / fc7 with dropout and loss_rcnn; the loss is rpn_loss + loss_rcnn.  Backward:
    the head and the RoI pooling into dfeat, split into a gradient activation; the RPN heads' and conv's weight gradients;
    the RPN conv's data gradient with the split dfeat added in its epilogue (frcnn_conv2d_res), so the feature map's two
    gradients meet without a pass of their own; then the trunk.  Each half is _RpnStep's and _RcnnStep's own code; the RPN
    half's head lives on `rpn` (_RpnNames).

    Flat layout: the trunk, the RPN 3x3 conv, fc6, fc7, cls_score | bbox_pred, then the RPN's twin heads; nothing is frozen
    and every step parameter lies after the trunk (VGG16's early exchange from conv4_1 covers only finished gradients)."""

    @property
    def _rpn(self):
        return self.rpn

    def _step_table(self, A):
        rpn_layers, rpn_params, _ = _RpnStep._step_table(self, A)
        _, rcnn_params, _ = _RcnnStep._step_table(self, A)
        return rpn_layers, rcnn_params + rpn_params, []

    def _joint_options(self, subsample, sample, dropout, post_n):
        """Raises FrcnnError for a bad one-image option (before anything is allocated)."""
        who = type(self).__name__
        if subsample not in ("device", "numpy", "none"):
            raise FrcnnError("%s: subsample must be one of ['device', 'none', 'numpy'] (got %r)" % (who, subsample))
        if sample != "numpy":
            raise FrcnnError("%s: sample must be 'numpy' (keep_inds= pins the kept rows) (got %r)" % (who, sample))
        if dropout not in (True, False):
            raise FrcnnError("%s: dropout must be True or False (masks= pins the masks) (got %r)" % (who, dropout))
        if not 1 <= int(post_n) <= 4096:
            raise FrcnnError("%s: post_n must be in [1, 4096] (got %r)" % (who, post_n))

    def _init_joint(self, params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                    loss_lambda, rpn_delta, subsample, num_classes, rcnn_delta, post_n, pre_n, nms_thresh, min_size, sample,
                    seed, dropout, optimizer=None):
        self._joint_options(subsample, sample, dropout, post_n)
        self.num_classes, self.rpn = num_classes, _RpnNames()
        self._init_common(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                          optimizer=optimizer)
        self._init_rpn_head(loss_lambda, rpn_delta, subsample, seed)
        self.rpn.targets = train_ops.AnchorTargets(self.A, self.fh, self.fw, self.device)
        self._init_rcnn_head(rcnn_delta, post_n, pre_n, nms_thresh, min_size)
        self._init_rcnn_draws(sample, seed, dropout)
        self.repack()

    def repack(self):
        self._repack_trunk()
        self._repack_rpn()
        self._repack_rcnn()

    # ---------------------------------------------------------------- forward
    def forward(self, x_chw, gt_boxes, im_info=None, disable_pos=None, keep_inds=None, masks=None):
        """x_chw (3,H,W) float32 CUDA; gt_boxes [G,5] float32 CUDA; disable_pos pins the RPN's subsampling, keep_inds the
        kept rows and masks the dropout masks, as in RpnTrainer / RcnnTrainer.  Returns losses float32[8] (device):
        rpn_loss_cls, rpn_loss_bbox, rpn_cls_accuracy, rpn_loss, loss_cls, loss_bbox, cls_accuracy, loss_rcnn."""
        im_h, im_w = (self.H, self.W) if im_info is None else (int(im_info[0]), int(im_info[1]))
        feat = self._forward_trunk(x_chw)
        self._rpn_trained_forward(feat)
        rpn = self._rpn_losses(gt_boxes, im_h, im_w, disable_pos)
        rcnn = self._rcnn_losses(feat, self.rpn.head_out, self.rpn.head_ld, gt_boxes, im_h, im_w, keep_inds, masks)
        self.last_losses = torch.cat([rpn, rcnn])
        return self.last_losses

    # ---------------------------------------------------------------- backward
    def backward(self, debug=None):
        """Fills g_flat with d(rpn_loss + loss_rcnn)/d(parameter): the RPN's parameters from rpn_loss, the head's from
        loss_rcnn, the trunk's from both.  debug: RcnnTrainer's head entries ("heads", "fc7", "fc6", "roi"), RpnTrainer's
        RPN entries with the twin heads under "RPN/heads" ("RPN/rpn_conv_3x3"'s "g_out" is the joined gradient of the
        feature map), and the trunk's."""
        dfeat = self._backward_rcnn(debug)
        self._backward_trunk(self._backward_rpn(debug, res=dfeat, tag=JOIN_TAG), debug)

    def step(self, x_chw, gt_boxes, im_info=None, disable_pos=None, keep_inds=None, masks=None):
        losses = self.forward(x_chw, gt_boxes, im_info, disable_pos, keep_inds, masks)
        self.backward()
        self.update()
        return losses


class _CanvasSteps(object):
    """The canvas machinery shared by _CanvasRpnStep and _CanvasRcnnStep: the N-slot image input with its device extents,
    the staged ground truth, the launches over the canvas (the _ext convolutions, zero outside each image, and the _batch
    re-layouts) that override _ConvTrainer's, and the capture-then-replay step."""
    raw_input = False           # True: the input is RawPhotoInput's training block (put_raw / step_raw)
    augment = None              # "device" | "list": the step draws or reads each slot's flip and scale (raw input only)
    level_ext = None            # the ResNet trunk's per-level extents int32 [5, N, 2] (None: the VGG16 trunk's halvings)

    def _canvas_options(self, N, max_gt):
        """Raises FrcnnError for a bad slot count or max_gt (before anything is allocated)."""
        who = type(self).__name__
        if int(N) != N or N < 1:
            raise FrcnnError("%s needs N >= 1 slots (got %r)" % (who, N))
        if int(max_gt) < 1:
            raise FrcnnError("%s: max_gt must be at least 1" % who)

    def _augment_options(self, raw_input, augment, scales, flip):
        """Raises FrcnnError for a bad augmentation (before anything is allocated)."""
        who = type(self).__name__
        if augment not in (None, "device", "list"):
            raise FrcnnError("%s: augment must be None, 'device' or 'list' (got %r)" % (who, augment))
        if augment is None:
            if tuple(scales) != (600,) or not flip:
                raise FrcnnError("%s: scales and flip need augment='device' or 'list'" % who)
            return
        if not raw_input:
            raise FrcnnError("%s: augment=%r needs raw_input=True (the float input is augmented by the caller)" % (who, augment))
        scales = tuple(scales)
        if not 1 <= len(scales) <= preprocess.AUG_MAX_SCALES or any(int(v) != v or v < 1 for v in scales):
            raise FrcnnError("%s: scales must be 1 to %d positive integers (got %r)" % (who, preprocess.AUG_MAX_SCALES, scales))

    def _canvas_init(self, N, Hc, Wc, max_gt, seed, raw_input, augment=None, scales=(600,), flip=True):
        dev = self.device
        self.raw_input = bool(raw_input)
        self.augment, self.flip = augment, bool(flip)
        self.scales = tuple(int(v) for v in scales)
        self._candidates = []                   # the staged photos' candidate im_scale (augment)
        self.input = (RawPhotoInput(N, Hc, Wc, dev, max_gt=max_gt, scales=self.scales if augment else None) if self.raw_input
                      else ImageInput(N, Hc, Wc, dev, canvas=True))
        self.x_in, self.extents, self.im_info = self.input.x_in, self.input.extents, self.input.im_info
        self.gt = torch.zeros((N, max_gt, 5), dtype=torch.float32, device=dev)
        self.gt_counts = torch.zeros((N,), dtype=torch.int32, device=dev)
        self.seeds = torch.arange(N, dtype=torch.int64, device=dev) + int(seed)
        self.image_sizes = [(0, 0)] * N
        self.graph = None

    # ---------------------------------------------------------------- launches over the canvas
    def _level(self, at):
        """(extents, halvings) of the trunk level `at`: the image extents and `at` halvings on the VGG16 trunk; on the ResNet
        trunk, whose levels are not ceil(e / 2^k) (pool1 is (c - 2) / 2 + 1), level `at` of level_ext with halvings 0."""
        if self.level_ext is None:
            return self.extents, at
        return self.level_ext[at], 0

    def _conv(self, x, planes, bias, ksize, relu, at, **kw):
        """frcnn_conv2d_batch_ext over the trunk level's extents, or over the head's (1, R_n) for "rois" / "roi_grads"."""
        ext, k = (self.head_ext, 0) if at in ("rois", "roi_grads") else self._level(at)
        return ops.conv2d_batch(x, planes[0], planes[1], bias, ksize, relu, extents=ext, halvings=k, **kw)

    def _prep(self, h, w, c, **kw):
        train_ops.grad_prepare_batch(self.N, h, w, c, **kw)

    def _pool(self, y, out):
        ops.maxpool2x2_ceil_batch(y, out=out)

    def _res_conv(self, x, planes, bias, ksize, relu, res, at, out):
        ext, k = self._level(at)
        ops.conv2d_res_batch(x, planes[0], planes[1], bias, ksize, relu, res, out=out, extents=ext, halvings=k)

    def _pool3(self, y, out, at):
        ops.maxpool3x3s2_ceil_batch(y, out=out, extents=self._level(at)[0])

    def _subsample(self, x, out):
        ops.subsample2x_batch(x, out=out)          # 0 outside each image, as its input is

    def _pool3_backward(self, g, y, p, out, tbuf):
        train_ops.maxpool3x3s2_backward_batch(self.N, g, y, p, out=out, tbuf=tbuf)

    def _prep_stride2(self, h, w, c, g, y, out, tbuf):
        train_ops.grad_prepare_stride2_batch(self.N, h, w, c, g, y=y, out=out, tbuf=tbuf)

    def _chw(self, act):
        """[N, C, H, W] float32 copy of an [N, H, W, C] Act (debug)."""
        return torch.stack([ops.Act(act.hi[n], None if act.lo is None else act.lo[n]).to_chw_f32() for n in range(self.N)])

    def _pack_input(self, x_chw=None):
        """The staged slots into x_col; raw photos are resized on the way, and their boxes scaled into gt.  On the ResNet
        trunk the first launch derives every level's extents from the staged sizes, so a captured step re-derives them.  An
        augmenting step first selects each slot's flip and scale (frcnn_voc_augment_batch: drawn from the step's seeds in
        "device" mode, as put_raw staged them in "list" mode), so every later launch reads the augmented sizes."""
        if self.augment is not None:
            self.input.augment(self.seeds, 0 if self.augment == "list" else (1 if self.flip else 2))
        if self.level_ext is not None:
            ops.resnet_level_extents(self.extents, self.H, self.W, out=self.level_ext)
        self.input.pack_im2col(self.x_col, *self.first_layer)
        if self.raw_input:
            self.input.scale_gt(self.gt, self.gt_counts)

    # ---------------------------------------------------------------- staging
    def _need_input(self, call):
        """Raises FrcnnError when `call` ("put" or "put_raw") does not match the input the trainer was built with."""
        if self.raw_input != (call == "put_raw"):
            raise FrcnnError("%s.%s: the trainer was built with raw_input=%s, so it takes %s" % (
                type(self).__name__, call, self.raw_input, "raw photos through put_raw / step_raw" if self.raw_input
                else "float images through put / step"))

    def _check_gt(self, images, gt_boxes):
        who = type(self).__name__
        if len(gt_boxes) != len(images):
            raise FrcnnError("%s.put: %d images and %d ground-truth lists" % (who, len(images), len(gt_boxes)))
        for n, g in enumerate(gt_boxes):
            if g.dim() != 2 or g.shape[1] != 5 or not 1 <= g.shape[0] <= self.max_gt:
                raise FrcnnError("%s.put: image %d has ground truth of shape %s, needs (G, 5) with 1 <= G <= %d"
                                 % (who, n, tuple(g.shape), self.max_gt))

    def _stage(self, images, gt_boxes, img_infos):
        """Images (ImageInput.put raises before its first copy if one does not fit) and ground truth into the static buffers."""
        sizes = self.input.put(images, img_infos)
        self.image_sizes = [tuple(int(v) for v in e) for e in sizes[0]]
        counts = np.zeros((self.N,), dtype=np.int32)
        for n, g in enumerate(gt_boxes):
            counts[n] = g.shape[0]
            self.gt[n, :g.shape[0]].copy_(g, non_blocking=True)
        self.gt_counts.copy_(torch.from_numpy(counts), non_blocking=True)

    def _stage_raw(self, photos, boxes, labels, flips=None, scale_index=None):
        """Photos, boxes and labels into the raw block in one host-to-device copy (RawPhotoInput.upload raises before it if
        something does not fit); the first launch of the step resizes them and scales the boxes.  Returns [im_scale] (with
        augment: each photo's tuple of candidate im_scale).  flips / scale_index: the choice of an augment="list" trainer."""
        who = type(self).__name__
        if (flips is not None or scale_index is not None) and self.augment != "list":
            raise FrcnnError("%s.put_raw: flips and scale_index need augment='list' (the trainer has %r)" % (who, self.augment))
        if flips is not None and not self.flip and any(flips):
            raise FrcnnError("%s.put_raw: the trainer was built with flip=False" % who)
        preprocess.raw_photo_shapes(photos)
        hdr, scales = self.input.upload(photos, boxes=list(boxes), labels=list(labels), flips=flips, scale_index=scale_index)
        if self.augment is None:
            self.image_sizes = [tuple(int(v) for v in e) for e in preprocess.raw_header_views(hdr, self.N)["extents"]]
        else:
            self._candidates = scales
            self.image_sizes = None
            if self.augment == "list":
                k = [0] * len(photos) if scale_index is None else [int(v) for v in scale_index]
                sizes = [preprocess.plan_size(x.shape[0], x.shape[1], self.scales[k[n]])[1:] for n, x in enumerate(photos)]
                self.image_sizes = sizes + [(0, 0)] * (self.N - len(photos))
        return scales

    def augmentation(self):
        """Each slot's (flip, im_scale, (H, W)) in the last step that ran on the photos put_raw staged last, in one download
        ((False, 0.0, (0, 0)) for an empty slot); it also sets image_sizes, which an augment="device" trainer leaves None
        after put_raw.  Raises FrcnnError on a trainer built without augment."""
        if self.augment is None:
            raise FrcnnError("%s.augmentation: the trainer was built without augment" % type(self).__name__)
        inp = self.input
        host = inp.block[:inp.header_bytes].cpu().numpy()
        views = preprocess.raw_header_views(host, self.N)
        aug_at = inp.header_bytes - preprocess.voc_aug_layout(self.N, len(self.scales))[1]
        aug = preprocess.voc_aug_views(host[aug_at:], self.N, len(self.scales))
        out = []
        for n in range(self.N):
            H, W = (int(v) for v in views["extents"][n])
            if n >= len(self._candidates) or H == 0:
                out.append((False, 0.0, (0, 0)))
                continue
            k = min(max(int(aug["choice"][n, 1]), 0), len(self.scales) - 1)
            out.append((bool(aug["flip"][n]), self._candidates[n][k], (H, W)))
        self.image_sizes = [o[2] for o in out]
        return out

    @staticmethod
    def _stage_lists(lists, N, buf, offsets):
        """Per-image int32 lists into one flat device buffer + offsets [N+1] (slots without a list get an empty range)."""
        lens = np.zeros((N,), dtype=np.int64)
        lens[:len(lists or [])] = [int(d.numel()) for d in lists or []]
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        for n, d in enumerate(lists or []):
            if lens[n]:
                buf[offs[n]:offs[n + 1]].copy_(d.reshape(-1), non_blocking=True)
        offsets.copy_(torch.from_numpy(offs), non_blocking=True)

    # ---------------------------------------------------------------- the step
    def _advance_seeds(self):
        """The step's last draw-related launch: when the step draws from its seeds (the step's _draws), slot n's seed moves
        on by N, once per step, so that slot n of step t draws with seed + t*N + n."""
        if self._draws():
            self.seeds.add_(self.N)

    def run(self):
        """Enqueues forward + backward + update on the current stream, with no host synchronisation."""
        self.forward()
        self.backward()
        self.update()

    def _step(self):
        """run() on what put() staged.  In a single process the first call runs eagerly (which also sets up every kernel's
        lazy state) and captures run() into a CUDA graph that every later call replays; with a process group of more than
        one rank the step stays eager, so the gradient exchange is not captured.  Returns the per-slot losses, float32
        [N, 4] on the device."""
        if self._multi():
            self.run()
        elif self.graph is None:
            self.run()
            losses = self.step_losses.clone()
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            self._capturing = True                   # the hyper-parameters are written before each replay, not captured
            try:
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    self.run()
            finally:
                self._capturing = False
            self.n_updates -= 1                      # the capture ran nothing
            self.graph = g
            return losses
        else:
            self._write_hyper()
            self.graph.replay()
            self.n_updates += 1
        return self.step_losses.clone()


class _CanvasRpnStep(_CanvasSteps, _RpnStep):
    """_RpnStep on a canvas (CanvasRpnTrainer describes it): staging, the batched anchor targets and loss."""

    _MODES = {"device": train_ops.SUBSAMPLE_DEVICE, "list": train_ops.SUBSAMPLE_LIST, "none": train_ops.SUBSAMPLE_NONE}

    def _init_canvas_rpn(self, params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, loss_lambda,
                         delta, subsample, seed, max_gt, device, process_group, raw_input, optimizer=None, augment=None,
                         scales=(600,), flip=True):
        """Checks the options, then builds the trunk, the RPN head, the canvas input, the batched anchor targets and the
        subsampling lists; then the first repack."""
        self._canvas_options(N, max_gt)
        self._augment_options(raw_input, augment, scales, flip)
        self._subsample_options(subsample)
        self.N, self.max_gt = N, max_gt = int(N), int(max_gt)
        self._init_common(params, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                          lead=(N,), optimizer=optimizer)
        self._init_rpn_head(loss_lambda, delta, subsample, seed)
        self._canvas_init(N, Hc, Wc, max_gt, seed, raw_input, augment, scales, flip)
        self._init_canvas_rpn_targets()
        self.step_losses = self.targets.losses
        self.repack()

    def _subsample_options(self, subsample):
        if subsample not in self._MODES:
            raise FrcnnError("%s: subsample must be one of %s" % (type(self).__name__, sorted(self._MODES)))

    def _init_canvas_rpn_targets(self):
        """The batched anchor targets, the twin heads' gradient and the subsampling lists."""
        r, N, dev = self._rpn, self.N, self.device
        r.head_grad = torch.empty_like(r.head_out)     # every element written by frcnn_rpn_loss_batch
        r.targets = train_ops.AnchorTargetsBatch(N, self.A, self.fh, self.fw, self.max_gt, dev)
        self.disable_pos = torch.zeros((max(N * r.targets.cap, 1),), dtype=torch.int32, device=dev)
        self.disable_offsets = torch.zeros((N + 1,), dtype=torch.int32, device=dev)

    # ---------------------------------------------------------------- staging
    def put(self, images, gt_boxes, img_infos=None, disable_pos=None):
        """Stages up to N (3,H_n,W_n) float32 CUDA images, their [G_n,5] ground-truth boxes (1 <= G_n <= max_gt), optional
        clip bounds (default (H_n, W_n)) and, in "list" mode, optional per-image disable lists into the static buffers
        (the remaining slots are empty).  Raises FrcnnError before anything is queued when something does not fit."""
        self._need_input("put")
        images, gt_boxes = list(images), list(gt_boxes)
        self._check_gt(images, gt_boxes)
        disable_pos = self._check_disable("put", len(images), disable_pos)
        self._stage(images, gt_boxes, img_infos)
        if self.subsample == "list":
            self._stage_lists(disable_pos, self.N, self.disable_pos, self.disable_offsets)

    def put_raw(self, photos, boxes, labels, disable_pos=None, flips=None, scale_index=None):
        """put() for a trainer built with raw_input=True: up to N raw uint8 (h, w, 3) BGR photos (numpy), their boxes (G_n, 4)
        in source-photo coordinates and labels (G_n,), 1 <= G_n <= max_gt, uploaded in one host-to-device copy.  The step
        applies the VOC training dataset's transform on the device: mean subtraction, the bicubic resize of
        preprocess.plan_size (short side 600, long side at most 1000), boxes times float32 im_scale; the clip bounds are the
        resized (H_n, W_n).  Raises FrcnnError before anything is queued when something does not fit.  Returns [im_scale].

        With augment, each photo is first mirrored (p[:, ::-1], boxes flipped in its w0 columns) when its flip is set, and
        resized at its chosen short side among `scales`; every candidate must fit the canvas.  "device": the step draws both
        from its seeds; "list": flips [bool] and scale_index [int] per photo (default no flip, index 0).  Returns each
        photo's tuple of candidate im_scale."""
        self._need_input("put_raw")
        photos = list(photos)
        disable_pos = self._check_disable("put_raw", len(photos), disable_pos)
        scales = self._stage_raw(photos, boxes, labels, flips, scale_index)
        if self.subsample == "list":
            self._stage_lists(disable_pos, self.N, self.disable_pos, self.disable_offsets)
        return scales

    def _check_disable(self, call, n_images, disable_pos):
        who = type(self).__name__
        if disable_pos is not None:
            disable_pos = list(disable_pos)
            if self.subsample != "list":
                raise FrcnnError("%s.%s: disable lists need subsample='list' (the trainer has %r)" % (who, call, self.subsample))
            if len(disable_pos) != n_images:
                raise FrcnnError("%s.%s: %d images and %d disable lists" % (who, call, n_images, len(disable_pos)))
            cap = self._rpn.targets.cap
            if any(int(d.numel()) > cap for d in disable_pos):
                raise FrcnnError("%s.%s: a disable list is longer than %d anchors" % (who, call, cap))
        return disable_pos

    # ---------------------------------------------------------------- forward
    def forward(self):
        """Forward over the staged canvas, the anchor targets and the per-slot losses (float32 [N, 4] device buffer:
        rpn_loss_cls, rpn_loss_bbox, rpn_cls_accuracy, rpn_loss; zeros for an empty slot)."""
        self._rpn_trained_forward(self._forward_trunk())
        self.last_losses = self._rpn_losses_batch()
        self._advance_seeds()
        return self.last_losses

    def _rpn_losses_batch(self):
        """The batched anchor targets and rpn_loss on _rpn.head_out, with the step's seeds; fills _rpn.head_grad.  Returns
        the per-slot losses, float32 [N, 4]."""
        (ext, k), r = self._level(self.halvings), self._rpn
        train_ops.anchor_targets_batch(self.anchors, self.A, self.feat_stride, ext, self.im_info, self.gt, self.gt_counts,
                                       r.targets, halvings=k, mode=self._MODES[self.subsample], seeds=self.seeds,
                                       disable_pos=self.disable_pos, disable_offsets=self.disable_offsets)
        return train_ops.rpn_loss_batch(r.head_out, r.head_ld, self.anchors, self.A, self.feat_stride, ext, self.im_info,
                                        r.targets, halvings=k, delta=r.delta, loss_lambda=self.loss_lambda, dhead=r.head_grad)

    def _draws(self):
        return self.subsample == "device" or self.augment == "device"

    def step(self, images, gt_boxes, img_infos=None, disable_pos=None):
        """put() + run(), captured into a CUDA graph after the first call (_CanvasSteps._step).  Returns the per-slot
        losses, float32 [N, 4] on the device."""
        self.put(images, gt_boxes, img_infos, disable_pos)
        return self._step()

    def step_raw(self, photos, boxes, labels, disable_pos=None, flips=None, scale_index=None):
        """put_raw() + run(), captured like step().  Returns the per-slot losses, float32 [N, 4] on the device."""
        self.put_raw(photos, boxes, labels, disable_pos, flips, scale_index)
        return self._step()


class _CanvasRcnnStep(_CanvasSteps, _RcnnStep):
    """_RcnnStep on a canvas (CanvasRcnnTrainer describes it): staging, device-side sampling and dropout, the batched
    proposals, targets, RoI pooling and loss."""

    _SAMPLE = {"device": train_ops.SUBSAMPLE_DEVICE, "list": train_ops.SUBSAMPLE_LIST}
    _DROPOUT = ("device", "explicit", None)

    def _init_canvas_rcnn(self, params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, num_classes,
                          delta, post_n, pre_n, nms_thresh, min_size, sample, dropout, seed, max_gt, device, process_group,
                          raw_input, optimizer=None, augment=None, scales=(600,), flip=True):
        """Checks the options, then builds the trunk, the canvas input, the frozen RPN and the head, the batched proposals,
        targets, kept lists and masks; then the first repack."""
        self._canvas_options(N, max_gt)
        self._augment_options(raw_input, augment, scales, flip)
        self._sampling_options(sample, dropout, post_n)
        self.N, self.max_gt = N, max_gt = int(N), int(max_gt)
        self.num_classes = num_classes
        self._init_common(params, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                          lead=(N,), optimizer=optimizer)
        self._canvas_init(N, Hc, Wc, max_gt, seed, raw_input, augment, scales, flip)
        self._frozen_rpn(params)
        self._init_rcnn_head(delta, post_n, pre_n, nms_thresh, min_size)
        self._init_canvas_rcnn_targets(sample, dropout)
        self.step_losses = self.ptargets.losses
        self.repack()

    def _sampling_options(self, sample, dropout, post_n):
        who = type(self).__name__
        if sample not in self._SAMPLE:
            raise FrcnnError("%s: sample must be one of %s" % (who, sorted(self._SAMPLE)))
        if dropout not in self._DROPOUT:
            raise FrcnnError("%s: dropout must be one of %s" % (who, self._DROPOUT))
        if not 1 <= int(post_n) <= 4096:
            raise FrcnnError("%s: post_n must be in [1, 4096] (got %r)" % (who, post_n))

    def _init_canvas_rcnn_targets(self, sample, dropout):
        """The head's extents, the batched proposals, targets, kept lists and masks, the head's gradient and the RoI
        pooling backward's workspace."""
        self.sample, self.dropout = sample, dropout
        N, nc, pre_n, post_n = self.N, self.num_classes, self.pre_n, self.post_n
        dev, fh, fw = self.device, self.fh, self.fw
        # the head's extents (1, R_n): column 1 is the proposal count frcnn_proposals_batch_ext writes
        self.head_ext = torch.ones((N, 2), dtype=torch.int32, device=dev)
        self.prop = ops.ProposalBatchWorkspace(N, self.A, fh, fw, pre_n, post_n, dev, outputs=(
            torch.zeros((N, post_n, 4), dtype=torch.float32, device=dev), torch.zeros((N, post_n), dtype=torch.float32, device=dev),
            self.head_ext[:, 1]))
        self.ptargets = train_ops.ProposalTargetsBatch(N, post_n, nc, dev)
        self.keep_list = torch.zeros((N * train_ops.ROIS_PER_IMAGE,), dtype=torch.int32, device=dev)
        self.keep_offsets = torch.zeros((N + 1,), dtype=torch.int32, device=dev)
        self.masks = torch.zeros((2, N, post_n, 4096), dtype=torch.uint8, device=dev) if dropout is not None else None
        self.head_grad = torch.empty_like(self.head_out)     # every element written by frcnn_rcnn_loss_batch
        self.roi_ws = torch.empty((ops._lib.load().frcnn_roi_pool_backward_batch_workspace_bytes(N, fh, fw, self.feat_ch),),
                                  dtype=torch.uint8, device=dev)

    # ---------------------------------------------------------------- staging
    def put(self, images, gt_boxes, img_infos=None, keep_inds=None, masks=None):
        """Stages up to N (3,H_n,W_n) float32 CUDA images with their [G_n,5] ground truth (1 <= G_n <= max_gt) and optional
        clip bounds; in "list" mode optional per-image kept lists (int, at most 128 distinct rows each; a slot without one
        keeps nothing), with dropout "explicit" per-image (fc6, fc7) uint8 [post_n, 4096] masks (a slot without masks keeps
        nothing).  Raises FrcnnError before anything is queued when something does not fit."""
        self._need_input("put")
        images, gt_boxes = list(images), list(gt_boxes)
        self._check_gt(images, gt_boxes)
        keep_inds, masks = self._check_extras("put", len(images), keep_inds, masks)
        self._stage(images, gt_boxes, img_infos)
        self._stage_extras(keep_inds, masks)

    def put_raw(self, photos, boxes, labels, keep_inds=None, masks=None, flips=None, scale_index=None):
        """put() for a trainer built with raw_input=True: raw photos, boxes and labels (and with augment="list" the flips and
        scale indices) as CanvasRpnTrainer.put_raw takes them, with put()'s kept lists and masks.  Returns [im_scale] (with
        augment: each photo's candidate im_scale tuple)."""
        self._need_input("put_raw")
        photos = list(photos)
        keep_inds, masks = self._check_extras("put_raw", len(photos), keep_inds, masks)
        scales = self._stage_raw(photos, boxes, labels, flips, scale_index)
        self._stage_extras(keep_inds, masks)
        return scales

    def _check_extras(self, call, n_images, keep_inds, masks):
        who = type(self).__name__
        if keep_inds is not None:
            keep_inds = [torch.as_tensor(k).reshape(-1) for k in keep_inds]
            if self.sample != "list":
                raise FrcnnError("%s.%s: kept lists need sample='list' (the trainer has %r)" % (who, call, self.sample))
            if len(keep_inds) != n_images:
                raise FrcnnError("%s.%s: %d images and %d kept lists" % (who, call, n_images, len(keep_inds)))
            for n, k in enumerate(keep_inds):
                if k.numel() > train_ops.ROIS_PER_IMAGE:
                    raise FrcnnError("%s.%s: image %d keeps %d rows, at most %d"
                                     % (who, call, n, k.numel(), train_ops.ROIS_PER_IMAGE))
                if torch.unique(k).numel() != k.numel():
                    raise FrcnnError("%s.%s: image %d's kept list repeats a row" % (who, call, n))
            keep_inds = [k.to(device=self.device, dtype=torch.int32) for k in keep_inds]
        if masks is not None:
            masks = list(masks)
            if self.dropout != "explicit":
                raise FrcnnError("%s.%s: masks need dropout='explicit' (the trainer has %r)" % (who, call, self.dropout))
            if len(masks) != n_images:
                raise FrcnnError("%s.%s: %d images and %d mask pairs" % (who, call, n_images, len(masks)))
            want = (self.post_n, 4096)
            for n, pair in enumerate(masks):
                if len(pair) != 2 or any(tuple(m.shape) not in (want, (want[0] * want[1],)) or m.dtype != torch.uint8 for m in pair):
                    raise FrcnnError("%s.%s: image %d needs two uint8 %s masks" % (who, call, n, want))
        return keep_inds, masks

    def _stage_extras(self, keep_inds, masks):
        if self.sample == "list":
            self._stage_lists(keep_inds, self.N, self.keep_list, self.keep_offsets)
        if self.dropout == "explicit":
            self.masks.zero_()
            for n, pair in enumerate(masks or []):
                for j in range(2):
                    self.masks[j, n].copy_(pair[j].reshape(self.post_n, 4096), non_blocking=True)

    # ---------------------------------------------------------------- forward
    def forward(self):
        """Forward over the staged canvas, the proposal targets and the per-slot losses (float32 [N, 4] device buffer:
        loss_cls, loss_bbox, cls_accuracy, loss_rcnn; zeros for a slot that kept nothing)."""
        feat = self._forward_trunk()
        self._rpn_forward(feat, self.rpn3, self.rpn_heads, self.rpn_mid, self.rpn_ld, self.rpn_out)
        self.last_losses = self._rcnn_losses_batch(feat, self.rpn_out, self.rpn_ld)
        self._advance_seeds()
        return self.last_losses

    def _rcnn_losses_batch(self, feat, rpn_out, rpn_ld):
        """The batched ProposalLayer on an RPN's output (fp32 [N*fh*fw, rpn_ld]), proposal targets, RoI pooling, dropout
        masks, the head and its losses, with the step's seeds; fills head_grad.  Returns the per-slot losses, float32
        [N, 4]."""
        N, (ext, k), R_cap = self.N, self._level(self.halvings), self.post_n
        ops.proposals_batch(rpn_out.view(N, self.fh * self.fw, rpn_ld), None, self.anchors, self.A, self.fh, self.fw,
                            self.feat_stride, 0, 0, self.min_size, self.pre_n, R_cap, self.nms_thresh, layout="nhwc",
                            ld=rpn_ld, cls_is_logits=True, work=self.prop, extents=ext, halvings=k, im_info=self.im_info)
        rois, count = self.prop.rois, self.head_ext[:, 1]
        train_ops.proposal_targets_batch(rois, count, self.gt, self.gt_counts, self.ptargets, mode=self._SAMPLE[self.sample],
                                         seeds=self.seeds, keep_list=self.keep_list, list_offsets=self.keep_offsets)
        p5 = ops.Act(self.pool5.hi.view(N, R_cap, -1), None if self.pool5.lo is None else self.pool5.lo.view(N, R_cap, -1))
        ops.roi_pool_batch(feat, rois, count, 7, 7, 1.0 / self.feat_stride, out=p5, extents=ext, halvings=k)
        if self.dropout == "device":
            for j in range(2):
                train_ops.dropout_masks_batch(self.seeds, j + 1, self.masks[j])
        self._head_forward()
        return train_ops.rcnn_loss_batch(self.head_out, self.ptargets, delta=self.delta, dhead=self.head_grad)

    def _draws(self):
        return self.sample == "device" or self.dropout == "device" or self.augment == "device"

    def _roi_pool_backward(self, g):
        ext, k = self._level(self.halvings)
        train_ops.roi_pool_backward_batch(self.feat, self.prop.rois, self.head_ext[:, 1], g, ext, k, 7, 7, 1.0 / self.feat_stride,
                                          out=self.dfeat, ws=self.roi_ws)

    def step(self, images, gt_boxes, img_infos=None, keep_inds=None, masks=None):
        """put() + run(), captured into a CUDA graph after the first call (_CanvasSteps._step).  Returns the per-slot
        losses, float32 [N, 4] on the device."""
        self.put(images, gt_boxes, img_infos, keep_inds, masks)
        return self._step()

    def step_raw(self, photos, boxes, labels, keep_inds=None, masks=None, flips=None, scale_index=None):
        """put_raw() + run(), captured like step().  Returns the per-slot losses, float32 [N, 4] on the device."""
        self.put_raw(photos, boxes, labels, keep_inds, masks, flips, scale_index)
        return self._step()


class _CanvasJointStep(_CanvasRpnStep, _CanvasRcnnStep, _JointStep):
    """_JointStep on a canvas (CanvasJointTrainer describes it): _CanvasRpnStep's anchor targets and loss and
    _CanvasRcnnStep's proposals, targets, RoI pooling and loss on the one RPN output, with both steps' staging."""

    def _init_canvas_joint(self, params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, loss_lambda,
                           rpn_delta, subsample, num_classes, rcnn_delta, post_n, pre_n, nms_thresh, min_size, sample, dropout,
                           seed, max_gt, device, process_group, raw_input, optimizer=None, augment=None, scales=(600,),
                           flip=True):
        """Checks both steps' options, then builds the trunk, the RPN head, the canvas input, the head, both steps'
        batched targets and lists; then the first repack."""
        self._canvas_options(N, max_gt)
        self._augment_options(raw_input, augment, scales, flip)
        self._subsample_options(subsample)
        self._sampling_options(sample, dropout, post_n)
        self.N, self.max_gt = N, max_gt = int(N), int(max_gt)
        self.num_classes, self.rpn = num_classes, _RpnNames()
        self._init_common(params, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                          lead=(N,), optimizer=optimizer)
        self._init_rpn_head(loss_lambda, rpn_delta, subsample, seed)
        self._canvas_init(N, Hc, Wc, max_gt, seed, raw_input, augment, scales, flip)
        self._init_rcnn_head(rcnn_delta, post_n, pre_n, nms_thresh, min_size)
        self._init_canvas_rpn_targets()
        self._init_canvas_rcnn_targets(sample, dropout)
        self.repack()

    @property
    def step_losses(self):
        """The last step's per-slot losses, float32 [N, 8]: the RPN step's four, then the RCNN step's."""
        return torch.cat([self.rpn.targets.losses, self.ptargets.losses], dim=1)

    # ---------------------------------------------------------------- staging
    def put(self, images, gt_boxes, img_infos=None, disable_pos=None, keep_inds=None, masks=None):
        """Stages up to N images with their ground truth and clip bounds, as CanvasRpnTrainer.put, with both steps' pins:
        disable lists (subsample="list"), kept lists (sample="list") and masks (dropout="explicit").  Raises FrcnnError
        before anything is queued when something does not fit."""
        self._need_input("put")
        images, gt_boxes = list(images), list(gt_boxes)
        self._check_gt(images, gt_boxes)
        disable_pos = self._check_disable("put", len(images), disable_pos)
        keep_inds, masks = self._check_extras("put", len(images), keep_inds, masks)
        self._stage(images, gt_boxes, img_infos)
        self._stage_pins(disable_pos, keep_inds, masks)

    def put_raw(self, photos, boxes, labels, disable_pos=None, keep_inds=None, masks=None, flips=None, scale_index=None):
        """put() for a trainer built with raw_input=True, as CanvasRpnTrainer.put_raw.  Returns [im_scale] (with augment:
        each photo's candidate im_scale tuple)."""
        self._need_input("put_raw")
        photos = list(photos)
        disable_pos = self._check_disable("put_raw", len(photos), disable_pos)
        keep_inds, masks = self._check_extras("put_raw", len(photos), keep_inds, masks)
        scales = self._stage_raw(photos, boxes, labels, flips, scale_index)
        self._stage_pins(disable_pos, keep_inds, masks)
        return scales

    def _stage_pins(self, disable_pos, keep_inds, masks):
        if self.subsample == "list":
            self._stage_lists(disable_pos, self.N, self.disable_pos, self.disable_offsets)
        self._stage_extras(keep_inds, masks)

    # ---------------------------------------------------------------- forward
    def forward(self):
        """Forward over the staged canvas and both steps' per-slot losses, float32 [N, 8] (step_losses)."""
        feat = self._forward_trunk()
        self._rpn_trained_forward(feat)
        self._rpn_losses_batch()
        self._rcnn_losses_batch(feat, self.rpn.head_out, self.rpn.head_ld)
        self._advance_seeds()
        self.last_losses = self.step_losses
        return self.last_losses

    def _draws(self):
        return _CanvasRpnStep._draws(self) or _CanvasRcnnStep._draws(self)

    def step(self, images, gt_boxes, img_infos=None, disable_pos=None, keep_inds=None, masks=None):
        """put() + run(), captured into a CUDA graph after the first call (_CanvasSteps._step).  Returns the per-slot
        losses, float32 [N, 8] on the device."""
        self.put(images, gt_boxes, img_infos, disable_pos, keep_inds, masks)
        return self._step()

    def step_raw(self, photos, boxes, labels, disable_pos=None, keep_inds=None, masks=None, flips=None, scale_index=None):
        """put_raw() + run(), captured like step().  Returns the per-slot losses, float32 [N, 8] on the device."""
        self.put_raw(photos, boxes, labels, disable_pos, keep_inds, masks, flips, scale_index)
        return self._step()


class RpnTrainer(_Vgg16Trunk, _RpnStep):
    """Weights, optimizer state and buffers of the RPN-mode training step for one image shape."""

    def __init__(self, params, H, W, anchors, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=16, loss_lambda=1.0, delta=3.0, subsample="device", seed=0, device="cuda", process_group=None,
                 optimizer=None):
        self._init_rpn(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                       loss_lambda, delta, subsample, seed, optimizer=optimizer)


class RcnnTrainer(_Vgg16Trunk, _RcnnStep):
    """One train_rcnn.py step (`model.rcnn_train = True`, /root/reference models/faster_rcnn.py:114-173): trunk -> RPN in TEST
    mode (its weights are frozen here: proposals are plain arrays, faster_rcnn.py:117-120) -> ProposalTargetLayer ->
    RoI pooling of ALL proposals -> fc6 / fc7 with dropout -> cls_score | bbox_pred -> losses on the kept rows ->
    backward through the head, the RoI pooling and the 13 trunk convolutions -> WeightDecay + MomentumSGD.
    Trainable: trunk/*, fc6, fc7, cls_score, bbox_pred (the RPN links receive no gradient: cleargrads semantics).

    fc6/W is kept internally in the (h, w, c) input order the RoI-pool kernel emits (`export_params` converts back).
    Sampling (`sample="numpy"`): the proposals' best overlaps come back to the host and np.random.choice draws exactly as
    proposal_target_layer.py:99-129 does, so a seeded run reproduces the reference's kept set; `keep_inds=` pins it.
    Dropout masks are explicit inputs (uint8 [post_n, 4096] x 2) or drawn from a torch generator."""

    def __init__(self, params, H, W, anchors, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=16, num_classes=21, delta=1.0, post_n=300, pre_n=6000, nms_thresh=0.7, min_size=16,
                 sample="numpy", seed=0, dropout=True, device="cuda", process_group=None, optimizer=None):
        self._init_rcnn(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                        num_classes, delta, post_n, pre_n, nms_thresh, min_size, sample, seed, dropout, optimizer=optimizer)


class CanvasRpnTrainer(_Vgg16Trunk, _CanvasRpnStep):
    """The RPN-mode training step on N images of different sizes per update, with one set of weights and optimizer state.

    Each image sits at the top-left of its slot of an N-slot Hc x Wc canvas (engine.ImageInput); its size and clip bounds
    are device arrays that every launch reads at run time, so one trainer -- and one captured CUDA graph -- serves any mix
    of sizes up to the canvas.  Forward and backward are RpnTrainer's chain over [N]-slabs: the *_batch_ext convolutions
    (zero outside each image), frcnn_anchor_targets_batch / frcnn_rpn_loss_batch (slot n is normalised by its own counts
    and anchor count, like the reference's per-device loss), frcnn_grad_prepare_batch and weight-gradient GEMMs over
    K = N*Kp, so the gradient is the SUM of the N per-image gradients (ParallelUpdater's addgrads, train_rpn.py:169-174),
    followed by one WeightDecay + MomentumSGD update.  Inside each image every activation, masked gradient and data
    gradient equals RpnTrainer's on that image alone, bit for bit; with N = 1 and an image that fills the canvas the whole
    step does.

    subsample "device": slot n of step t draws with seed + t*N + n (a device counter advanced inside the step, so a replayed
    graph draws fresh samples): the k-th image of a stream gets the labels RpnTrainer(seed=seed) gives its k-th image.
    "list": put() takes per-image disable lists (positions in the inside-compact order, frcnn_anchor_targets mode 2).
    "none": labels before subsampling.

    augment (raw_input=True only; None keeps the plain VOC transform): "device" draws each slot's horizontal flip and
    short side among `scales` on the device from the step's seed (seed + t*N + n, salt 3), so a replayed graph augments
    afresh; "list" takes them from put_raw(flips=, scale_index=).  flip=False jitters the scale only.  augmentation()
    downloads what the last step chose."""

    def __init__(self, params, N, Hc, Wc, anchors, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=16, loss_lambda=1.0, delta=3.0, subsample="device", seed=0, max_gt=256, device="cuda",
                 process_group=None, raw_input=False, optimizer=None, augment=None, scales=(600,), flip=True):
        self._init_canvas_rpn(params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, loss_lambda,
                              delta, subsample, seed, max_gt, device, process_group, raw_input, optimizer=optimizer,
                              augment=augment, scales=scales, flip=flip)


class CanvasRcnnTrainer(_Vgg16Trunk, _CanvasRcnnStep):
    """The RCNN-mode training step (RcnnTrainer's, train_rcnn.py) on N images of different sizes per update, with one set of
    weights and optimizer state and one captured CUDA graph.

    Forward: the canvas trunk, the frozen RPN (_ext convolutions + frcnn_proposals_batch_ext, whose per-slot proposal count
    is written straight into column 1 of the [N][2] extents (1, R_n) of the head), frcnn_proposal_targets_batch,
    frcnn_roi_pool_batch_ext, fc6 / fc7 / cls_score | bbox_pred as _ext convolutions over N x 1 x R_cap (rows >= R_n are 0,
    as RcnnTrainer's m_valid leaves them), dropout, frcnn_rcnn_loss_batch (slot n normalised by its own kept count).
    Backward: the head and fc layers through frcnn_grad_prepare_batch with weight GEMMs over K = N*Kp,
    frcnn_roi_pool_backward_batch_ext, then the trunk; one WeightDecay + MomentumSGD update on the summed gradient.
    Inside each image every activation and data gradient equals RcnnTrainer's on that image with the same kept rows and
    masks, bit for bit.

    sample "device": slot n of step t samples with seed + t*N + n (frcnn_proposal_targets_batch mode 1, a device counter
    advanced inside the step); "list": put() takes per-image kept lists (RcnnTrainer's keep_inds, at most 128 distinct rows).
    dropout "device": masks drawn by frcnn_dropout_masks_batch from the same per-slot seeds (salt 1: fc6, 2: fc7); "explicit":
    put() takes per-image (fc6, fc7) uint8 [post_n, 4096] masks; None: no dropout.  `masks` [2, N, post_n, 4096] holds the
    masks the last step used.  augment / scales / flip: as CanvasRpnTrainer's; the draw shares the step's seed advance with
    the sampling and the dropout."""

    def __init__(self, params, N, Hc, Wc, anchors, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=16, num_classes=21, delta=1.0, post_n=300, pre_n=6000, nms_thresh=0.7, min_size=16,
                 sample="device", dropout="device", seed=0, max_gt=256, device="cuda", process_group=None, raw_input=False,
                 optimizer=None, augment=None, scales=(600,), flip=True):
        self._init_canvas_rcnn(params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, num_classes,
                               delta, post_n, pre_n, nms_thresh, min_size, sample, dropout, seed, max_gt, device,
                               process_group, raw_input, optimizer=optimizer, augment=augment, scales=scales, flip=flip)


class JointTrainer(_Vgg16Trunk, _JointStep):
    """One approximate-joint-training step (py-faster-rcnn's end2end recipe; the four losses the reference's train.py
    reports together): trunk -> the trained RPN, once -> AnchorTargetLayer + rpn_loss, and ProposalLayer on the same logits
    -> ProposalTargetLayer -> RoI pooling -> fc6 / fc7 with dropout -> cls_score | bbox_pred -> loss_rcnn; backward of
    rpn_loss + loss_rcnn (the RPN's parameters from rpn_loss, the head's from loss_rcnn, the trunk's from both; no gradient
    through the proposals' coordinates) -> WeightDecay + the optimizer's rule on every parameter.  export_params() is a
    whole detector, which Engine loads.

    The arguments are RpnTrainer's and RcnnTrainer's, rpn_delta and rcnn_delta being their two deltas.  Draws: the RPN's
    subsampling as RpnTrainer's (its seed counter, or NumPy's global RNG with subsample="numpy"), the kept rows as
    RcnnTrainer's (NumPy, after the RPN's draws) and the masks from a torch generator seeded with `seed`; disable_pos,
    keep_inds and masks pin them.  The proposal counts default to RcnnTrainer's test-mode ones; pass pre_n=12000,
    post_n=2000 for py-faster-rcnn's training counts."""

    def __init__(self, params, H, W, anchors, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=16, loss_lambda=1.0, rpn_delta=3.0, subsample="device", num_classes=21, rcnn_delta=1.0,
                 post_n=300, pre_n=6000, nms_thresh=0.7, min_size=16, sample="numpy", seed=0, dropout=True, device="cuda",
                 process_group=None, optimizer=None):
        self._init_joint(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                         loss_lambda, rpn_delta, subsample, num_classes, rcnn_delta, post_n, pre_n, nms_thresh, min_size,
                         sample, seed, dropout, optimizer=optimizer)


class CanvasJointTrainer(_Vgg16Trunk, _CanvasJointStep):
    """JointTrainer's step on N images of different sizes per update, with one set of weights and optimizer state and one
    captured CUDA graph (a multi-rank run stays eager, with the trunk's gradient exchange).

    The forward is CanvasRpnTrainer's trunk and RPN, run once, its batched anchor targets and loss, then
    CanvasRcnnTrainer's batched proposals (on the same RPN output), targets, RoI pooling, head and loss; the backward is
    the head's, then the RPN's with the split dfeat added in the RPN conv's data gradient, then the trunk's.  The gradient
    is the sum over the slots.  Inside each image everything equals JointTrainer's on that image alone with the same draws.
    Per-slot losses, float32 [N, 8]: the RPN's four, then the RCNN's.

    Draws: slot n of step t uses seed + t*N + n for the anchor subsampling, the RoI sampling, both dropout masks and the
    augmentation, and the step advances the seeds once, so step 0 draws the labels CanvasRpnTrainer(seed=seed) draws and the
    kept rows and masks CanvasRcnnTrainer(seed=seed) draws on the same proposals.  subsample / sample / dropout / augment
    and their pins (disable_pos, keep_inds, masks, flips, scale_index) are those two trainers'."""

    def __init__(self, params, N, Hc, Wc, anchors, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=16, loss_lambda=1.0, rpn_delta=3.0, subsample="device", num_classes=21, rcnn_delta=1.0,
                 post_n=300, pre_n=6000, nms_thresh=0.7, min_size=16, sample="device", dropout="device", seed=0, max_gt=256,
                 device="cuda", process_group=None, raw_input=False, optimizer=None, augment=None, scales=(600,), flip=True):
        self._init_canvas_joint(params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, loss_lambda,
                                rpn_delta, subsample, num_classes, rcnn_delta, post_n, pre_n, nms_thresh, min_size, sample,
                                dropout, seed, max_gt, device, process_group, raw_input, optimizer=optimizer, augment=augment,
                                scales=scales, flip=flip)
