"""models.faster_rcnn.FasterRCNN -- same class, constructor, train switches, side outputs and call
signature as /root/reference models/faster_rcnn.py:19-178, inference branch (:92-134,175-178):

    cls_prob, pred_boxes = model(x, img_info)      # Variable (R,21) softmax, ndarray (R,84) boxes

The whole graph (trunk -> RPN -> ProposalLayer -> RoI pool -> fc6/fc7 -> cls/bbox -> softmax/decode/
clip) is frcnn_b200.engine: hand-written sm_100a kernels behind the C ABI, replayed as ONE CUDA graph
per image shape.  Link names / parameter paths are the reference's, so `serializers.load_npz` of a
reference checkpoint (forward.py:29) fills this model.  RPN training mode (:114-116) returns rpn_loss computed on the
device (targets + losses + head gradient, models/region_proposal_network.py); RCNN training mode (:117-173) returns
loss_rcnn from frcnn_b200.train_engine.RcnnTrainer, or resnet_train.ResNetRcnnTrainer for a models.resnet.ResNet trunk
(kept in `self.rcnn_trainer` for backward / update).
"""
import os

from frcnn_b200 import arrays, links
from frcnn_b200.engine import Engine
from models.bbox_transform import bbox_transform_inv, clip_boxes  # noqa: F401  (reference import surface)
from models.region_proposal_network import RegionProposalNetwork
from models.vgg16 import VGG16


class FasterRCNN(links.Link):
    type_check_enable = int(os.environ.get('CHAINER_TYPE_CHECK', '1')) != 0
    precision = "bf16x3"        # "bf16": single-pass fast mode (not the parity mode)

    def __init__(self, trunk_class=VGG16, rpn_in_ch=512, rpn_mid_ch=512, feat_stride=16,
                 anchor_ratios=(0.5, 1, 2), anchor_scales=(8, 16, 32), num_classes=21, loss_lambda=1,
                 rpn_delta=3, rcnn_delta=1):
        super(FasterRCNN, self).__init__()
        self.add_link("trunk", trunk_class())
        self.add_link("RPN", RegionProposalNetwork(rpn_in_ch, rpn_mid_ch, feat_stride, anchor_ratios,
                                                   anchor_scales, num_classes, loss_lambda, rpn_delta))
        self.add_link("fc6", links.linear_link(rpn_in_ch * 7 * 7, 4096, 0.01))
        self.add_link("fc7", links.linear_link(4096, 4096, 0.01))
        self.add_link("cls_score", links.linear_link(4096, num_classes, 0.01))
        self.add_link("bbox_pred", links.linear_link(4096, num_classes * 4, 0.01))
        d = self.__dict__
        d["_feat_stride"], d["_anchor_ratios"], d["_anchor_scales"] = feat_stride, anchor_ratios, anchor_scales
        d["_num_classes"], d["_spatial_scale"] = num_classes, 1. / feat_stride
        d["_rpn_delta"], d["_rcnn_delta"] = rpn_delta, rcnn_delta
        d["_rcnn_train"] = False
        d["_engine"] = (None, -1)
        # forward.py:48-57 runs cpu_nms(dets, 0.3) per class on this call's host outputs (thresholds: forward.py:75-76).  With
        # a threshold here the inference graph runs that per-class NMS itself (frcnn_detect) and models.cpu_nms hands the
        # keep lists over when it is called on exactly those rows; None = the graph stops at (cls_prob, bbox_pred).
        d["caller_nms_thresh"], d["caller_nms_conf"] = 0.3, 0.8
        d["rpn_proposals"], d["rpn_probs"] = None, None
        self.RPN.train = False

    # -- train switches with the reference's coupling (:48-74)
    @property
    def rcnn_train(self):
        return self._rcnn_train

    @rcnn_train.setter
    def rcnn_train(self, val):
        self.__dict__["_rcnn_train"] = val
        if val:
            self.RPN.train = not val
        self.trunk.__dict__["train"] = bool(self.rcnn_train or self.rpn_train)

    @property
    def rpn_train(self):
        return self.RPN.train

    @rpn_train.setter
    def rpn_train(self, val):
        self.RPN.train = val
        if val:
            self.__dict__["_rcnn_train"] = not val
        self.trunk.__dict__["train"] = bool(self.rcnn_train or self.rpn_train)

    def _check_data_type_forward(self, x, img_info, gt_boxes):
        from chainer import Variable
        assert isinstance(x, Variable) and isinstance(img_info, Variable)
        assert x.shape[0] == 1 and arrays.dtype_kind(x) == 'f'
        assert img_info.shape == (1, 2) and arrays.dtype_kind(img_info) == 'i'
        if gt_boxes is not None:
            assert isinstance(gt_boxes, Variable)
            assert gt_boxes.shape[0] == 1 and gt_boxes.shape[1] > 0 and gt_boxes.shape[2] == 5
            assert arrays.dtype_kind(gt_boxes) == 'f'

    # -- parameters learnt by the device-side trainer flow back into the Link params before anyone reads them
    def _sync_trained_params(self):
        tr = self.__dict__.get("rcnn_trainer")
        if tr is None or self.__dict__.get("_rcnn_synced_updates", 0) == tr.n_updates:
            return
        named = dict(links.Link.namedparams(self))
        for k, v in tr.export_params().items():              # fc6/W comes back in the reference's (c, h, w) column order
            named["/" + k]._data[...] = v
        self._params_changed()
        self.__dict__["_rcnn_synced_updates"] = tr.n_updates
        shape_key = self.__dict__.get("_rcnn_trainer_key")
        if shape_key is not None:                              # the trainer already holds these weights: keep it
            self.__dict__["_rcnn_trainer_key"] = (shape_key[0], self.version_key())

    def namedparams(self, prefix=""):
        """serializers.save_npz / param_dict / the inference engine all read the parameters through here."""
        self._sync_trained_params()
        return links.Link.namedparams(self, prefix)

    def engine(self):
        eng, ver = self._engine
        n_layers = getattr(self.trunk, "n_layers", None)
        handoff = self.caller_nms_thresh if n_layers is None else None
        key = (self.version_key(), handoff, self.caller_nms_conf)
        if eng is None or ver != key:
            params = self.param_dict()
            kw = dict(precision=self.precision, anchors=self.RPN.proposal_layer._anchors, num_classes=self._num_classes,
                      n_anchors=self.RPN.proposal_layer._num_anchors, feat_stride=self._feat_stride)
            if handoff is not None:
                kw.update(with_detect=True, det_nms_thresh=float(handoff), det_conf=float(self.caller_nms_conf))
            if n_layers is not None:                    # models.resnet.ResNet trunk (SURVEY.md 8f rank 2)
                from frcnn_b200.resnet_engine import ResNetEngine
                eng = ResNetEngine(params, n_layers, **kw)
            else:
                eng = Engine(params, **kw)
            self.__dict__["_engine"] = (eng, key)
        return eng

    def __call__(self, x, img_info, gt_boxes=None):
        """x (1,3,H,W) preprocessed image, img_info (1,2) = (height, width) as the caller passes it
        (forward.py:93 passes (H, H), Q7) -> (Variable softmax (R,num_classes), pred_boxes (R,4*num_classes))."""
        from chainer import Variable
        if self.type_check_enable:
            self._check_data_type_forward(x, img_info, gt_boxes)
        if self.rpn_train and gt_boxes is not None:
            # RPN training mode (:114-116): trunk features -> RPN -> AnchorTargetLayer -> rpn_loss (a Variable); the
            # gradient w.r.t. the RPN head outputs is left in self.RPN.head_grad.  The backward pass through the convs
            # and the optimizer step are the remaining part of this "next" row.
            return self.RPN(self.trunk(x), img_info, gt_boxes)
        if gt_boxes is not None and self.rcnn_train:
            # RCNN training mode (:117-173): frozen test-mode RPN -> ProposalTargetLayer (NumPy-RNG sampling like the
            # reference) -> RoI pool -> fc6/fc7 with dropout -> losses on the kept rows, all in frcnn_b200.train_engine.
            # The trainer (weights, stored activations) is kept in self.rcnn_trainer: .backward() / .update() complete the
            # train_rcnn.py step; loss_cls / cls_accuracy / loss_bbox are attributes like the reference's reports.
            from frcnn_b200.resnet_train import ResNetRcnnTrainer
            from frcnn_b200.train_engine import RcnnTrainer
            fam = arrays.family(x)
            t = arrays.to_device(x)
            hw = arrays.to_host_ints(img_info)
            pl = self.RPN.proposal_layer
            tr = self.__dict__.get("rcnn_trainer")
            self._sync_trained_params()                       # weights a previous trainer learnt -> the Link params
            key = (tuple(t.shape[2:]), self.version_key())
            if tr is None or self.__dict__.get("_rcnn_trainer_key") != key:
                # a new image shape (VOC images vary in size) or externally changed parameters: the new trainer starts from
                # the CURRENT parameters (synced above) and inherits the optimizer, weight decay and optimizer state of the
                # one it replaces
                old = tr
                kw = dict(precision=self.precision, feat_stride=self._feat_stride, num_classes=self._num_classes,
                          delta=float(self._rcnn_delta), post_n=pl._post_nms_top_n, pre_n=pl._pre_nms_top_n,
                          nms_thresh=pl._nms_thresh, min_size=pl._min_size, device=t.device)
                if old is not None:
                    kw.update(optimizer=old.optimizer, weight_decay=old.weight_decay)
                n_layers = getattr(self.trunk, "n_layers", None)
                if n_layers is not None:                # models.resnet.ResNet trunk: frozen BatchNorm, as engine() runs it
                    tr = ResNetRcnnTrainer(self.param_dict(), int(t.shape[2]), int(t.shape[3]), pl._anchors, n_layers=n_layers,
                                           **kw)
                else:
                    tr = RcnnTrainer(self.param_dict(), int(t.shape[2]), int(t.shape[3]), pl._anchors, **kw)
                if old is not None and old.index == tr.index:
                    tr.load_optimizer_state(old.optimizer_state(to_host=False))
                self.__dict__["rcnn_trainer"], self.__dict__["_rcnn_trainer_key"] = tr, key
                self.__dict__["_rcnn_synced_updates"] = tr.n_updates
            losses = tr.forward(t[0], arrays.to_device(gt_boxes)[0], im_info=(int(hw[0]), int(hw[1])))
            vals = list(losses.cpu().numpy()) if fam == arrays.NUMPY else [arrays.from_device(losses[i].clone(), fam) for i in range(4)]
            d = self.__dict__
            d["loss_cls"], d["loss_bbox"], d["cls_accuracy"], d["loss_rcnn"] = [Variable(v) for v in vals]
            return self.loss_rcnn
        fam = arrays.family(x)
        hw = arrays.to_host_ints(img_info)
        pl = self.RPN.proposal_layer
        kw = dict(pre_n=pl._pre_nms_top_n, post_n=pl._post_nms_top_n, nms_thresh=pl._nms_thresh, min_size=pl._min_size)
        if fam == arrays.NUMPY:
            # the reference's CPU-mode call (forward.py:88-94): a HOST float32 image in, host arrays out.  One pinned
            # upload, the graph, ONE download of the whole result block; thread-safe (a plan per calling thread).
            import numpy as np
            xd = arrays.raw(x)
            if xd.dtype != np.float32:
                xd = xd.astype(np.float32)
            res, plan = self.engine().call_host(xd[0], img_info=(int(hw[0]), int(hw[1])), **kw)
            self.__dict__["rpn_proposals"] = res["rois"].copy()
            self.__dict__["rpn_probs"] = res["scores"].reshape(-1, 1).copy()
            from models import cpu_nms as _caller_nms
            if plan.with_detect:                         # the caller's per-class NMS already ran in the graph: hand it over
                _caller_nms.publish(res["prob"], res["boxes"], res["keep_idx"], res["keep_count"], plan.det_nms_thresh)
            else:
                _caller_nms.withdraw()
            return Variable(res["prob"].copy()), res["boxes"].copy()
        t = arrays.to_device(x)
        prob, boxes, plan = self.engine()(t[0], img_info=(int(hw[0]), int(hw[1])), **kw)
        R = prob.shape[0]
        self.__dict__["rpn_proposals"] = arrays.from_device(plan.prop.rois[:R].clone(), fam)
        self.__dict__["rpn_probs"] = arrays.from_device(plan.prop.scores[:R].reshape(R, 1).clone(), fam)
        return Variable(arrays.from_device(prob.clone(), fam)), arrays.from_device(boxes.clone(), fam)
