"""CPU tests of the forward plans' host side: the VGG16 trunk schedule the plans, the C structs and the trainers share, the
float-canvas sizes and the raw-photo block staging, and the engine's plan cache keys."""
import threading

import numpy as np
import pytest

from frcnn_b200 import engine, preprocess
from frcnn_b200._lib import FrcnnError

POOLED = ("conv1_2", "conv2_2", "conv3_3", "conv4_3")


def _trunk_by_rule(H, W, fuse_pool):
    """(trunk_steps, activation shapes after acts[0], feature size) by the rule: VGG16_LAYERS in order, every 2x2 pool maps
    h -> (h + 1) // 2, in the producing conv's epilogue when fuse_pool, else as its own activation."""
    steps, acts, h, w = [], [], H, W
    for name, _, cout in [it for it in engine.VGG16_LAYERS if it != "pool"]:
        pooled = name in POOLED
        if pooled and fuse_pool:
            h, w = (h + 1) // 2, (w + 1) // 2
        acts.append((h, w, cout))
        steps.append((name, pooled and fuse_pool, pooled and not fuse_pool))
        if pooled and not fuse_pool:
            h, w = (h + 1) // 2, (w + 1) // 2
            acts.append((h, w, cout))
    return steps, acts, (h, w)


class _ShapePlan(engine._PlanBase):
    """_PlanBase's trunk allocation with every activation replaced by its shape."""

    def __init__(self, fuse_pool):
        self.fuse_pool = fuse_pool

    def _act(self, *shape):
        return shape


@pytest.mark.parametrize("fuse_pool", [True, False])
@pytest.mark.parametrize("H,W", [(600, 1000), (16, 16), (37, 53), (1, 1), (75, 125)])
def test_vgg16_schedule_reproduces_the_trunk(H, W, fuse_pool):
    steps, acts, feat = _trunk_by_rule(H, W, fuse_pool)
    sched, feat_hw = engine.vgg16_schedule(H, W, fuse_pool)
    assert feat_hw == feat
    assert [s[:3] for s in sched] == [it for it in engine.VGG16_LAYERS if it != "pool"]
    assert [s.halvings for s in sched] == [0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4]
    p = _ShapePlan(fuse_pool)
    assert p._alloc_trunk(H, W) == feat
    assert p.trunk_steps == steps and p.acts[1:] == acts
    assert p.acts[0] == (engine.ops._lib.load().frcnn_image_c8_elems(H, W),)
    if (H, W) == (600, 1000):
        assert feat == (38, 63)


def test_trainer_layer_table():
    from frcnn_b200 import train_engine
    assert train_engine.TRUNK == [
        ("conv1_1", 3, 64), ("conv1_2", 64, 64), ("conv2_1", 64, 128), ("conv2_2", 128, 128), ("conv3_1", 128, 256),
        ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512),
        ("conv5_1", 512, 512), ("conv5_2", 512, 512), ("conv5_3", 512, 512)]
    assert train_engine.POOL_AFTER == set(POOLED)


def test_canvas_sizes():
    shapes = [(3, 64, 96), (3, 17, 5)]
    got = preprocess.canvas_sizes(shapes, 3, 64, 96)
    assert got.dtype == np.int32 and got.shape == (2, 3, 2)
    assert got.tolist() == [[[64, 96], [17, 5], [0, 0]], [[64, 96], [17, 5], [0, 0]]]
    got = preprocess.canvas_sizes(shapes, 2, 64, 96, img_infos=[(64, 64), (17.0, 17)])
    assert got.tolist() == [[[64, 96], [17, 5]], [[64, 64], [17, 17]]]
    assert preprocess.canvas_sizes([], 2, 8, 8).tolist() == [[[0, 0], [0, 0]], [[0, 0], [0, 0]]]
    with pytest.raises(FrcnnError, match="slots"):
        preprocess.canvas_sizes(shapes * 2, 3, 64, 96)
    with pytest.raises(FrcnnError, match="img_infos"):
        preprocess.canvas_sizes(shapes, 3, 64, 96, img_infos=[(64, 96)])
    for bad in [(3, 65, 96), (3, 64, 97), (3, 0, 96), (3, 64, 0), (1, 64, 96), (64, 96), (1, 3, 64, 96)]:
        with pytest.raises(FrcnnError, match="canvas"):
            preprocess.canvas_sizes([shapes[0], bad], 3, 64, 96)


def _photo(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("N,shapes", [(4, [(300, 500), (333, 500), (375, 500), (7, 5)]), (5, [(31, 17), (300, 500)]), (2, [])])
def test_fill_raw_block(N, shapes):
    photos = [_photo(h, w, i) for i, (h, w) in enumerate(shapes)]
    if photos:
        photos[0] = np.asfortranarray(photos[0])               # a strided photo is copied as its C-order bytes
    hdr, _, used = preprocess.raw_batch_header(preprocess.raw_photo_shapes(photos), N, 1000, 1000, 1 << 22)
    buf = np.full((hdr.size + (1 << 22),), 0xAB, dtype=np.uint8)
    n = preprocess.fill_raw_block(buf, hdr, photos, N)
    assert n == hdr.size + used
    assert np.array_equal(buf[:hdr.size], hdr)
    offs = preprocess.raw_header_views(hdr, N)["src_off"]
    for k, x in enumerate(photos):
        o = hdr.size + int(offs[k])
        assert np.array_equal(buf[o:o + x.nbytes], np.ascontiguousarray(x).reshape(-1))
    assert (buf[n:] == 0xAB).all()
    with pytest.raises(FrcnnError, match="block"):
        preprocess.fill_raw_block(buf[:n - 1], hdr, photos, N)


def test_raw_photo_shapes():
    ok = _photo(3, 4, 0)
    assert preprocess.raw_photo_shapes([ok, _photo(5, 2, 1)]) == [(3, 4), (5, 2)]
    for bad in [ok.astype(np.float32), ok[:, :, 0], ok[:, :, :2], ok.reshape(-1), ok.tolist()]:
        with pytest.raises(FrcnnError, match="photo 1"):
            preprocess.raw_photo_shapes([ok, bad])


def test_input_buffers():
    """The two static inputs on a CPU device: a float canvas's put() fills the slots and the [2, N, 2] sizes that extents /
    im_info view; a raw input's header arrays are views into its block at raw_header_layout's offsets, with the default
    arena and means, and a non-positive arena is refused."""
    torch = pytest.importorskip("torch")
    same = engine.ImageInput(2, 8, 12, "cpu", hwc_memory=True)
    assert same.extents is None and same.im_info is None and same.hwc_memory and tuple(same.x_in.shape) == (2, 3, 8, 12)
    canvas = engine.ImageInput(3, 8, 12, "cpu", canvas=True)
    x = torch.arange(3 * 5 * 7, dtype=torch.float32).view(3, 5, 7)
    assert canvas.put([x], img_infos=[(5, 5)]).tolist() == [[[5, 7], [0, 0], [0, 0]], [[5, 5], [0, 0], [0, 0]]]
    assert canvas.extents.tolist() == [[5, 7], [0, 0], [0, 0]] and canvas.im_info.tolist() == [[5, 5], [0, 0], [0, 0]]
    assert torch.equal(canvas.x_in[0, :, :5, :7], x) and canvas.x_in[0, :, 5:].abs().sum() == 0 and canvas.x_in[1:].abs().sum() == 0
    raw = engine.RawPhotoInput(3, 600, 1000, "cpu")
    layout, hb = preprocess.raw_header_layout(3)
    assert raw.x_in is None and raw.header_bytes == hb and raw.arena_bytes == 3 * 3 * 600 * 1000
    assert raw.block.numel() == hb + raw.arena_bytes and raw.arena.data_ptr() == raw.block.data_ptr() + hb
    assert raw.pixel_means == tuple(float(v) for v in np.asarray(preprocess.PIXEL_MEANS).reshape(-1))
    hdr, _, _ = raw.header([(300, 500), (375, 500)], img_infos=[(600, 600), (600, 800)])
    raw.block[:hb] = torch.from_numpy(hdr)
    want = preprocess.raw_header_views(hdr, 3)
    for name, t in zip(("arena", "src_off", "src_hw", "inv_scale", "extents"), raw.descriptors):
        if name != "arena":
            assert t.data_ptr() == raw.block.data_ptr() + layout[name][0] and np.array_equal(t.numpy(), want[name]), name
    assert raw.extents.tolist() == [[600, 1000], [600, 800], [0, 0]] and raw.im_info.tolist() == [[600, 600], [600, 800], [0, 0]]
    assert engine.RawPhotoInput(1, 8, 8, "cpu", pixel_means=np.array([[1, 2, 3]]), arena_bytes=64).pixel_means == (1.0, 2.0, 3.0)
    for bad in (0, -5):
        with pytest.raises(FrcnnError, match="arena_bytes"):
            engine.RawPhotoInput(2, 8, 8, "cpu", arena_bytes=bad)


class _StubPlan(object):
    """Records its constructor arguments; clone() makes another one."""

    def __init__(self, *args, **kw):
        self.args, self.kw = args, kw

    def clone(self):
        return type(self)(*self.args, **self.kw)


class _StubWeightsMixin(object):
    plan_class = _StubPlan

    def _pack_weights(self, *args):
        return ("weights",) + args


def test_engine_plan_cache_keys(monkeypatch):
    monkeypatch.setattr(engine, "BatchPlan", _StubPlan)
    monkeypatch.setattr(engine, "CanvasBatchPlan", _StubPlan)

    class Eng(_StubWeightsMixin, engine.Engine):
        pass

    eng = Eng({}, "bf16", "cuda:1", anchors="A", with_detect=True, post_n=50)
    assert eng.weights == ("weights", {}, "bf16", "cuda:1", 21, 9)
    kw = (("post_n", 50), ("use_graph", False), ("with_detect", True))
    p = eng.plan(64, 96, use_graph=False)
    b = eng.batch_plan(2, 64, 96, use_graph=False)
    c = eng.canvas_plan(3, 128, 192, use_graph=False)
    assert eng.plans == {(64, 96, kw): p, ("batch", 2, 64, 96, kw): b, ("canvas", 3, 128, 192, kw): c}
    assert p.args == (eng.weights, 64, 96) and b.args == (eng.weights, 2, 64, 96) and c.args == (eng.weights, 3, 128, 192)
    assert p.kw == dict(anchors="A", feat_stride=16, post_n=50, use_graph=False, with_detect=True) == b.kw == c.kw
    assert eng.plan(64, 96, use_graph=False) is p and eng.plan(64, 96, use_graph=True) is not p
    # thread_plan checks out plan()'s entry first, then clones of it for other threads
    assert eng.thread_plan(64, 96, use_graph=False) is p and eng.thread_plan(64, 96, use_graph=False) is p
    other = []
    t = threading.Thread(target=lambda: other.append(eng.thread_plan(64, 96, use_graph=False)))
    t.start()
    t.join()
    assert isinstance(other[0], _StubPlan) and other[0] is not p and other[0].args == p.args
    assert len(eng.plans) == 4


def test_resnet_engine_plan_cache_keys():
    from frcnn_b200 import resnet_engine as re_
    assert re_.ResNetEngine.plan_class is re_.ResNetForwardPlan

    class Eng(_StubWeightsMixin, re_.ResNetEngine):
        pass

    eng = Eng({}, 50, anchors="A", post_n=100)
    assert eng.n_layers == 50 and eng.weights == ("weights", {}, "bf16x3", "cuda", 21, 9)
    p = eng.plan(150, 201)
    assert eng.plans == {(150, 201, (("post_n", 100),)): p}
    assert p.args == (eng.weights, 150, 201) and p.kw == dict(anchors="A", feat_stride=32, post_n=100)
    with pytest.raises(FrcnnError):
        eng.batch_plan(2, 64, 96)
    with pytest.raises(FrcnnError):
        eng.canvas_plan(2, 64, 96)
