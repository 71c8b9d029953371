#!/usr/bin/env python
"""Run the REFERENCE's own Python for the hot path (from /root/reference, unmodified files) in this
container and freeze what it produces as golden fixtures: tests/golden/ref_*.npz.

TEST INFRASTRUCTURE.  Needs /root/reference (build container only); the GPU box only reads the
committed .npz files.  `python scripts/make_ref_fixtures.py` regenerates every fixture
deterministically (fixed seeds, tie-free scores where the reference's sort order would otherwise be
unspecified).

What runs (all imported from /root/reference through the import hook below):
  lib/mnc_config.py                      cfg (real values, not restated)
  lib/transform/anchors.py               generate_anchors                        :38-102
  lib/transform/bbox_transform.py        bbox_transform_inv / clip_boxes / filter_small_boxes :64-130
  lib/pylayer/proposal_layer.py          ProposalLayer.setup/.forward (TEST)     :27-175
  lib/pylayer/stage_bridge_layer.py      StageBridgeLayer.setup/.forward (TEST)  :25-80, 237-255
  lib/pylayer/mask_layer.py              MaskLayer.setup/.forward (TEST)         :20-48, 95-102
  lib/nms/nms_wrapper.py                 nms                                     :13-21
  lib/nms/py_cpu_nms.py                  py_cpu_nms (stand-in body of gpu_nms, see below)
  lib/transform/mask_transform.py        gpu_mask_voting                         :213-286
  lib/utils/blob.py                      prep_im_for_blob / im_list_to_blob      :17-50
  tools/demo.py                          prepare_mnc_args / im_detect            :54-100
  lib/utils/bbox.pyx                     bbox_overlaps, cythonized unmodified -> oracle/_ref/cython_bbox.so

Environment shims (the reference is Python 2 / numpy 1.x; none of these touches its arithmetic):
  * import hook: modules under /root/reference are compiled after two SYNTAX-only source patches --
    py2 `print x` statements -> `print(x)` (only in error/debug branches, never executed here) and
    `.iteritems()` -> `.items()` (proposal_layer.py:173, stage_bridge_layer.py:78, mask_layer.py:46);
  * builtins.xrange = range; numpy.float/int/bool aliases (removed in numpy 1.24);
    yaml.load(s) defaults to SafeLoader (PyYAML >= 6 made Loader mandatory);
  * stub modules: `easydict` (attribute dict), `caffe` (Layer base holding param_str_ / phase, and
    a Blob with .data / .reshape), `matplotlib.pyplot` and `cPickle` (imported by demo.py /
    utils/vis_seg.py, unused on the path);
  * native extensions.  `gpu_nms.gpu_nms` and `nms.mv.mv` are CUDA functions and this container has
    no GPU.  The script binds RECORDING stand-ins with the .pyx signatures (gpu_nms.pyx:16-31,
    gpu_mv.pyx:13-31): gpu_nms computes its answer with the reference's own py_cpu_nms.py (same
    IoU arithmetic and `>`-suppression as nms_kernel.cu:24-32,71 -- asserted on the GPU below),
    mv with the C oracle; every call's inputs and outputs are stored in ref_native_calls.npz, and
    tests/test_ref_pin.py::test_recorded_native_calls_replay replays them on the GPU box through the
    reference's real `_nms` / `_mv` (oracle/_ref/libmnc_ref.so, compiled unmodified) and asserts
    bit-identical outputs.  So every fixture equals what the reference produces with its own CUDA
    extensions, by transitivity through a test that can fail.
  * numpy-version semantics.  Two expressions on the path change meaning between the numpy 1.x
    the reference ran on and the numpy 2 in this image:
      - mask_transform.py:266-267 `cur_weights / sum(cur_weights)`: builtin sum() over float32
        scalars accumulates in float64 under numpy 1.x (int 0 + float32 -> float64) and in
        float32 under numpy 2 (NEP 50).  Both variants are recorded: `*_np2` as run here, `*_np1`
        with a module-level `sum` that accumulates in float64 and returns a Python float.
      - demo.py:92-93 `rois[:, 1:5] / im_scales[0]` (float32 array / 0-d float64 array): float32
        division under numpy 1.x, float64 under numpy 2.  Recorded as run here (float64); the
        oracle reproduces it with numpy2=True and tests bound the numpy-1 variant to 1 ulp.
"""
import builtins
import ctypes
import importlib.machinery
import importlib.util
import os
import re
import sys
import types

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")
sys.dont_write_bytecode = True


# --------------------------------------------------------------------------- import machinery
_PRINT = re.compile(r"^(\s*)print (.+)$", re.M)


class _RefLoader(importlib.machinery.SourceFileLoader):
    patched = {}

    def source_to_code(self, data, path, *, _optimize=-1):
        src = importlib.util.decode_source(data)
        new, n1 = _PRINT.subn(r"\1print(\2)", src)
        n2 = new.count(".iteritems()")
        new = new.replace(".iteritems()", ".items()")
        if n1 or n2:
            _RefLoader.patched[os.path.relpath(path, REF)] = {"print": n1, "iteritems": n2}
        return compile(new, path, "exec", dont_inherit=True, optimize=_optimize)


def _ref_path_hook(path):
    if not os.path.abspath(path).startswith(REF):
        raise ImportError
    return importlib.machinery.FileFinder(
        path, (importlib.machinery.ExtensionFileLoader, importlib.machinery.EXTENSION_SUFFIXES),
        (_RefLoader, importlib.machinery.SOURCE_SUFFIXES))


def install_reference_environment(native_log):
    import yaml
    builtins.xrange = range
    for name, typ in (("float", float), ("int", int), ("bool", bool)):
        if not hasattr(np, name):
            setattr(np, name, typ)
    _yaml_load = yaml.load
    yaml.load = lambda s, Loader=yaml.SafeLoader: _yaml_load(s, Loader=Loader)

    # easydict
    class EasyDict(dict):
        def __init__(self, d=None, **kw):
            super().__init__()
            for k, v in dict(d or {}, **kw).items():
                self[k] = v

        def __setitem__(self, k, v):
            if isinstance(v, dict) and not isinstance(v, EasyDict):
                v = EasyDict(v)
            super().__setitem__(k, v)

        __setattr__ = __setitem__

        def __getattr__(self, k):
            try:
                return self[k]
            except KeyError:
                raise AttributeError(k)
    m = types.ModuleType("easydict")
    m.EasyDict = EasyDict
    sys.modules["easydict"] = m

    # caffe: python_layer.hpp:27-46 protocol
    caffe = types.ModuleType("caffe")

    class Layer(object):
        param_str_ = ""
        phase = "TEST"
    caffe.Layer = Layer
    caffe.TEST = "TEST"
    sys.modules["caffe"] = caffe

    mpl = types.ModuleType("matplotlib")
    plt = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot = plt
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.pyplot"] = plt
    import pickle
    sys.modules["cPickle"] = pickle                     # utils/vis_seg.py:9 (imported by demo.py)

    sys.path_hooks.insert(0, _ref_path_hook)
    sys.path_importer_cache.clear()
    sys.path.insert(0, os.path.join(REF, "tools"))
    sys.path.insert(0, os.path.join(REF, "lib"))
    sys.path.insert(0, os.path.join(REF, "lib", "nms"))   # py2 implicit relative imports of nms/

    # utils.cython_bbox: the reference's bbox.pyx, cythonized unmodified (oracle/Makefile ref)
    import utils  # noqa: F401  (reference package)
    so = os.path.join(ROOT, "oracle", "_ref", "cython_bbox.so")
    spec = importlib.util.spec_from_file_location("bbox", so)
    bbox = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bbox)
    sys.modules["utils.cython_bbox"] = bbox

    # native stand-ins (see module docstring)
    from py_cpu_nms import py_cpu_nms   # reference file lib/nms/py_cpu_nms.py

    def gpu_nms(dets, thresh, device_id=0):
        assert dets.dtype == np.float32 and dets.ndim == 2      # gpu_nms.pyx:16 typed argument
        keep = [int(i) for i in py_cpu_nms(dets, thresh)]
        native_log["nms"].append((dets.copy(), float(thresh), np.asarray(keep, np.int64)))
        return keep
    g = types.ModuleType("gpu_nms")
    g.gpu_nms = gpu_nms
    sys.modules["gpu_nms"] = g
    c = types.ModuleType("cpu_nms")
    c.cpu_nms = py_cpu_nms
    sys.modules["cpu_nms"] = c

    sys.path.insert(0, ROOT)
    from oracle import oracle as O

    def mv(all_boxes, all_masks, candidate_inds, candidate_start, candidate_weights, image_height,
           image_width, device_id=0):
        for a, dt, nd in ((all_boxes, np.float32, 2), (all_masks, np.float32, 4),
                          (candidate_inds, np.int32, 1), (candidate_start, np.int32, 1),
                          (candidate_weights, np.float32, 1)):      # gpu_mv.pyx:13-20 typed args
            assert a.dtype == dt and a.ndim == nd
        rm, rb = O.mv(all_boxes, all_masks, candidate_inds, candidate_start, candidate_weights,
                      int(image_height), int(image_width))
        native_log["mv"].append((all_boxes.copy(), all_masks.copy(), candidate_inds.copy(),
                                 candidate_start.copy(), candidate_weights.copy(),
                                 int(image_height), int(image_width), rm.copy(), rb.copy()))
        return rm, rb
    import nms  # noqa: F401  (reference package lib/nms)
    mvm = types.ModuleType("nms.mv")
    mvm.mv = mv
    sys.modules["nms.mv"] = mvm
    return caffe


class Blob(object):
    """bottom[i] / top[i] as pycaffe exposes them (_caffe.cpp:273-288): .data float32, .reshape."""

    def __init__(self, data=None):
        self.data = np.zeros((1,), np.float32) if data is None else np.ascontiguousarray(data, np.float32)

    def reshape(self, *dims):
        if tuple(dims) != self.data.shape:
            self.data = np.zeros(dims, np.float32)

    @property
    def shape(self):
        return self.data.shape


def tie_free_scores(rng, n, lo=0.001, hi=0.999):
    s = rng.permutation(np.linspace(lo, hi, n)).astype(np.float32)
    assert np.unique(s).size == n
    return s


def boxes_in_image(rng, n, W, H, smin=16, smax=400, cluster=0):
    """f32 boxes inside a WxH image; with `cluster`, jittered copies of n/cluster seeds so that
    IoU >= 0.5 groups exist (mask voting needs overlapping candidates)."""
    if cluster:
        seeds = boxes_in_image(rng, (n + cluster - 1) // cluster, W, H, smin, smax)
        b = np.repeat(seeds, cluster, axis=0)[:n] + rng.normal(0, 6, size=(n, 4)).astype(np.float32)
    else:
        cx = rng.uniform(0, W, n)
        cy = rng.uniform(0, H, n)
        w = np.exp(rng.uniform(np.log(smin), np.log(smax), n))
        h = np.exp(rng.uniform(np.log(smin), np.log(smax), n))
        b = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], 1)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, W - 1)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, H - 1)
    x1 = np.minimum(b[:, 0], b[:, 2]); x2 = np.maximum(b[:, 0], b[:, 2])
    y1 = np.minimum(b[:, 1], b[:, 3]); y2 = np.maximum(b[:, 1], b[:, 3])
    return np.stack([x1, y1, x2, y2], 1).astype(np.float32)


def softmax_rows(rng, n, c, scale=1.0):
    z = rng.normal(0, scale, size=(n, c))
    e = np.exp(z - z.max(1, keepdims=True))
    return (e / e.sum(1, keepdims=True)).astype(np.float32)


def save_parts(path, items, limit=900000):
    """np.savez_compressed in as many files as it takes to keep each under `limit` bytes:
    <name>.npz, <name>.part2.npz, ... (tests/test_ref_fixtures.py load() reads them back as one)."""
    import io

    def size(d):
        b = io.BytesIO()
        np.savez_compressed(b, **d)
        return len(b.getvalue())
    parts = [{}]
    for k, v in items.items():
        trial = dict(parts[-1])
        trial[k] = v
        if parts[-1] and size(trial) > limit:
            parts.append({k: v})
        else:
            parts[-1] = trial
    for i, d in enumerate(parts):
        np.savez_compressed(path if i == 0 else "%s.part%d.npz" % (path[:-4], i + 1), **d)


def main():
    native = {"nms": [], "mv": []}
    install_reference_environment(native)
    from mnc_config import cfg
    from transform.anchors import generate_anchors
    from transform.bbox_transform import bbox_transform_inv, clip_boxes, filter_small_boxes
    from pylayer.proposal_layer import ProposalLayer
    from pylayer.stage_bridge_layer import StageBridgeLayer
    from pylayer.mask_layer import MaskLayer
    import transform.mask_transform as mask_transform
    from utils.blob import prep_im_for_blob, im_list_to_blob
    from utils.cython_bbox import bbox_overlaps
    import demo

    os.makedirs(OUT, exist_ok=True)
    meta = {}

    def O_shifted_anchors(H, W):   # the anchor enumeration of proposal_layer.py:84-100, via the
        from oracle import oracle as O   # oracle (only used for the margin self-check below)
        return O.shifted_anchors(H, W, 16)

    # ---- cfg values the path reads (lib/mnc_config.py) ------------------------------------------
    cfgv = {
        "PIXEL_MEANS": cfg.PIXEL_MEANS, "BINARIZE_THRESH": cfg.BINARIZE_THRESH,
        "MASK_SIZE": cfg.MASK_SIZE, "TEST_SCALES": np.array(cfg.TEST.SCALES),
        "TRAIN_MAX_SIZE": cfg.TRAIN.MAX_SIZE, "TEST_MAX_SIZE": cfg.TEST.MAX_SIZE,
        "TEST_NMS": cfg.TEST.NMS, "RPN_NMS_THRESH": cfg.TEST.RPN_NMS_THRESH,
        "RPN_PRE_NMS_TOP_N": cfg.TEST.RPN_PRE_NMS_TOP_N,
        "RPN_POST_NMS_TOP_N": cfg.TEST.RPN_POST_NMS_TOP_N, "RPN_MIN_SIZE": cfg.TEST.RPN_MIN_SIZE,
        "MASK_MERGE_IOU_THRESH": cfg.TEST.MASK_MERGE_IOU_THRESH,
        "MASK_MERGE_NMS_THRESH": cfg.TEST.MASK_MERGE_NMS_THRESH,
        "USE_GPU_NMS": cfg.USE_GPU_NMS, "USE_GPU_MASK_MERGE": cfg.TEST.USE_GPU_MASK_MERGE,
    }
    np.savez_compressed(os.path.join(OUT, "ref_cfg.npz"), **{k: np.asarray(v) for k, v in cfgv.items()})

    # ---- anchors + bbox transforms ---------------------------------------------------------------
    rng = np.random.default_rng(101)
    bt = {"anchors": generate_anchors()}
    for tag, n, ncol, bdt in (("a", 500, 4, np.float64), ("b", 300, 84, np.float32)):
        boxes = boxes_in_image(rng, n, 1000, 600).astype(bdt)
        deltas = rng.normal(0, 0.6, size=(n, ncol)).astype(np.float32)
        pred = bbox_transform_inv(boxes, deltas)
        clipped, keep = clip_boxes(pred, np.array([600, 1000], np.float32))
        small = filter_small_boxes(clipped[:, :4], 16 * 1.6)
        bt.update({"boxes_" + tag: boxes, "deltas_" + tag: deltas, "pred_" + tag: pred,
                   "clipped_" + tag: clipped, "clip_keep_" + tag: keep, "small_keep_" + tag: small})
    bt["pred_empty"] = bbox_transform_inv(np.zeros((0, 4), np.float32), np.zeros((0, 84), np.float32))
    q = boxes_in_image(rng, 40, 1000, 600, cluster=4).astype(np.float64)
    bt["ov_boxes"] = q
    bt["ov"] = bbox_overlaps(q, q[::3].copy())
    np.savez_compressed(os.path.join(OUT, "ref_bbox.npz"), **bt)

    # ---- ProposalLayer.forward (TEST) ------------------------------------------------------------
    pl = {}
    cases = [("6x8", 6, 8, [96, 128, 1.0], 0.3, 201),
             ("38x63", 38, 63, [600, 1000, 1.0], 0.25, 202),          # configs[1] feature map
             ("38x50_s1.6", 38, 50, [600, 800, 1.6], 0.5, 203),      # scaled image: min_size 25.6
             ("19x32_wild", 19, 32, [300, 500, 0.8], 1.5, 204)]      # big deltas: clip + filter
    def proposal_margins(dets, deltas, H, W, im_info):
        """The CUDA path decodes with expf (<= 2 ulp from numpy's exp), so a fixture must not have a
        decision sitting inside that noise (1e-7 relative on coordinates): returns the smallest
        |IoU - thresh| among the NMS input and the smallest |side - min_size| over all proposals."""
        b64 = dets[:, :4].astype(np.float64)
        area = (b64[:, 2] - b64[:, 0] + 1) * (b64[:, 3] - b64[:, 1] + 1)
        worst = 1.0
        for s0 in range(0, len(b64), 500):
            c = b64[s0:s0 + 500]
            iw = np.minimum(c[:, None, 2], b64[None, :, 2]) - np.maximum(c[:, None, 0], b64[None, :, 0]) + 1
            ih = np.minimum(c[:, None, 3], b64[None, :, 3]) - np.maximum(c[:, None, 1], b64[None, :, 1]) + 1
            inter = np.clip(iw, 0, None) * np.clip(ih, 0, None)
            iou = inter / (area[s0:s0 + 500, None] + area[None, :] - inter)
            worst = min(worst, np.abs(iou - cfg.TEST.RPN_NMS_THRESH).min())
        pr_all, _ = clip_boxes(bbox_transform_inv(O_shifted_anchors(H, W),
                                                  deltas.transpose(0, 2, 3, 1).reshape(-1, 4)),
                               np.array(im_info[:2], np.float32))
        sides = np.concatenate([pr_all[:, 2] - pr_all[:, 0] + 1, pr_all[:, 3] - pr_all[:, 1] + 1])
        return float(worst), float(np.abs(sides - cfg.TEST.RPN_MIN_SIZE * np.float32(im_info[2])).min())

    for tag, H, W, im_info, dstd, seed in cases:
        for attempt in range(200):      # first seed (seed + 1000 k) whose margins are safe
            seed_used = seed + 1000 * attempt
            rng = np.random.default_rng(seed_used)
            A = 9
            fg = tie_free_scores(rng, A * H * W).reshape(1, A, H, W)
            prob = np.concatenate([1 - fg, fg], axis=1).astype(np.float32)
            deltas = rng.normal(0, dstd, size=(1, 4 * A, H, W)).astype(np.float32)
            layer = ProposalLayer()
            layer.param_str_ = "'feat_stride': 16"                      # test.prototxt:473
            layer.phase = "TEST"
            bottom = [Blob(prob), Blob(deltas), Blob(np.array([im_info], np.float32))]
            top = [Blob()]
            n0 = len(native["nms"])
            layer.setup(bottom, top)
            layer.reshape(bottom, top)
            layer.forward(bottom, top)
            assert len(native["nms"]) == n0 + 1
            m_iou, m_side = proposal_margins(native["nms"][-1][0], deltas, H, W, im_info)
            if m_iou > 2e-6 and m_side > 1e-3:
                meta["proposal_%s_margins" % tag] = [m_iou, m_side]
                meta["proposal_%s_seed" % tag] = seed_used
                break
            native["nms"].pop()
        else:
            raise AssertionError("no margin-safe seed for " + tag)
        pl.update({"prob_" + tag: prob, "deltas_" + tag: deltas,
                   "im_info_" + tag: np.array([im_info], np.float32), "rois_" + tag: top[0].data.copy(),
                   "ind_after_filter_" + tag: np.asarray(layer._ind_after_filter),
                   "ind_after_sort_" + tag: np.asarray(layer._ind_after_sort),
                   "proposal_index_" + tag: np.asarray(layer._proposal_index)})
        meta["proposal_" + tag] = int(top[0].data.shape[0])
    pl["cases"] = np.array([c[0] for c in cases])
    save_parts(os.path.join(OUT, "ref_proposal.npz"), pl)

    # ---- StageBridgeLayer / MaskLayer (TEST) -----------------------------------------------------
    sb = {}
    for tag, n, im_info, seed in (("a", 300, [600, 1000, 1.0], 301), ("b", 120, [600, 800, 1.6], 302)):
        rng = np.random.default_rng(seed)
        rois = np.hstack([np.zeros((n, 1), np.float32),
                          boxes_in_image(rng, n, im_info[1], im_info[0])]).astype(np.float32)
        bbox_pred = rng.normal(0, 0.25, size=(n, 84)).astype(np.float32)
        prob = softmax_rows(rng, n, 21, 2.0)
        prob[5, :] = 0.0; prob[5, 0] = 0.5; prob[5, 7] = 0.5        # tie: class 0 (bg) wins argmax
        prob[6, :] = 0.0; prob[6, 3] = 0.4; prob[6, 9] = 0.4        # tie: first max (3)
        layer = StageBridgeLayer()
        layer.param_str_ = "{'feat_stride': 16, 'use_clip': 1, 'clip_base': 512, 'num_classes': 21}"
        layer.phase = "TEST"
        bottom = [Blob(rois), Blob(bbox_pred), Blob(prob), Blob(np.array([im_info], np.float32))]
        top = [Blob()]
        layer.setup(bottom, top)
        layer.reshape(bottom, top)
        layer.forward(bottom, top)
        sb.update({"rois_" + tag: rois, "bbox_pred_" + tag: bbox_pred, "prob_" + tag: prob,
                   "im_info_" + tag: np.array([im_info], np.float32), "rois_ext_" + tag: top[0].data.copy()})
    rng = np.random.default_rng(303)
    mo = rng.uniform(0, 1, size=(7, 441)).astype(np.float32)
    layer = MaskLayer()
    layer.phase = "TEST"
    top = [Blob()]
    layer.setup([Blob(mo)], top)
    layer.forward([Blob(mo)], top)
    sb["mask_output"] = mo
    sb["mask_proposal"] = top[0].data.copy()
    np.savez_compressed(os.path.join(OUT, "ref_stage_bridge.npz"), **sb)

    # ---- gpu_mask_voting -------------------------------------------------------------------------
    def sum_np1(xs):
        t = np.float64(0.0)
        for v in xs:
            t = t + np.float64(v)
        return float(t)

    mvf = {}
    vcases = [("a", 600, 1000, 600, 4, 401), ("b", 300, 500, 375, 6, 402), ("c", 90, 320, 224, 3, 403)]
    for tag, nb, W, H, cluster, seed in vcases:
        rng = np.random.default_rng(seed)
        boxes = boxes_in_image(rng, nb, W, H, 24, 300, cluster=cluster)
        # mask values k/4096 (exact in fp32; stored as uint16 so the fixture stays small)
        mask_q = np.clip(np.round(4096.0 / (1.0 + np.exp(-rng.normal(0, 2, size=(nb, 1, 21, 21))))),
                         1, 4095).astype(np.uint16)
        masks = (mask_q.astype(np.float32) / np.float32(4096.0)).astype(np.float32)
        scores = softmax_rows(rng, nb, 21, 2.5)
        assert all(np.unique(scores[:, c]).size == nb for c in range(1, 21))   # tie-free per class
        for variant in ("np2", "np1"):
            if variant == "np1":
                mask_transform.sum = sum_np1
            elif "sum" in mask_transform.__dict__:
                del mask_transform.sum
            n0 = len(native["mv"])
            lm, lb = mask_transform.gpu_mask_voting(masks, boxes, scores, 21, 100, W, H)
            assert len(native["mv"]) == n0 + 1
            call = native["mv"][-1]
            mvf.update({"cand_inds_%s_%s" % (tag, variant): call[2], "cand_start_%s_%s" % (tag, variant): call[3],
                        "cand_weights_%s_%s" % (tag, variant): call[4],
                        "class_counts_%s_%s" % (tag, variant): np.array([len(b) for b in lb], np.int32),
                        "result_box_%s_%s" % (tag, variant): np.vstack(lb),
                        "result_mask_%s_%s" % (tag, variant): np.concatenate(lm, 0)})
        if "sum" in mask_transform.__dict__:
            del mask_transform.sum
        mvf.update({"boxes_" + tag: boxes, "masks_q4096_" + tag: mask_q, "scores_" + tag: scores,
                    "hw_" + tag: np.array([H, W])})
        # the 20 per-class NMS calls of this case (identical in both variants): keep lists only,
        # dets = hstack(boxes, scores[:, c]) is rebuilt by the replay test
        calls = native["nms"][-40:-20]
        for c, (dets, thr, keep) in enumerate(calls, start=1):
            assert thr == cfg.TEST.MASK_MERGE_NMS_THRESH
            assert np.array_equal(dets, np.hstack((boxes, scores[:, c:c + 1])))
            mvf["nms_keep_%s_c%d" % (tag, c)] = keep.astype(np.int32)
        meta["voting_" + tag] = int(sum(len(b) for b in lb))
    save_parts(os.path.join(OUT, "ref_voting.npz"), mvf)

    # ---- prep_im_for_blob / prepare_mnc_args / im_detect tail -----------------------------------
    class Net(object):
        def __init__(self, blobs):
            self.blobs = blobs
            self.fed = None

        def forward(self, **kw):
            self.fed = kw
            return {}

    pr = {}
    pcases = (("150x200", 150, 200, 501), ("250x166", 250, 166, 502),     # scale 4.0, 3.614...
              ("600x1000", 600, 1000, 503), ("120x400", 120, 400, 504))   # scale 1.0; max-size cap 2.5
    for tag, H, W, seed in pcases:
        rng = np.random.default_rng(seed)
        # the image is rebuilt from its seed by the tests (PCG64 `integers` stream; crc guards it)
        im = np.random.default_rng(seed).integers(0, 256, size=(H, W, 3), dtype=np.uint8)
        n = 40
        blob_probe, scale = prep_im_for_blob(im.copy(), cfg.PIXEL_MEANS, cfg.TEST.SCALES[0], cfg.TRAIN.MAX_SIZE)
        sh, sw = blob_probe.shape[:2]
        blobs = {
            "data": Blob(), "im_info": Blob(),
            "rois": Blob(np.hstack([np.zeros((n, 1), np.float32), boxes_in_image(rng, n, sw, sh)])),
            "rois_ext": Blob(np.hstack([np.zeros((n, 1), np.float32), boxes_in_image(rng, n, sw, sh)])),
            "mask_proposal": Blob(rng.uniform(0, 1, size=(n, 1, 21, 21))),
            "mask_proposal_ext": Blob(rng.uniform(0, 1, size=(n, 1, 21, 21))),
            "seg_cls_prob": Blob(softmax_rows(rng, n, 21)),
            "seg_cls_prob_ext": Blob(softmax_rows(rng, n, 21)),
        }
        # make a few boxes touch / exceed the ORIGINAL image border after un-scaling
        blobs["rois"].data[0, 1:5] = [0, 0, sw - 1, sh - 1]
        blobs["rois_ext"].data[1, 1:5] = [sw - 1.2, sh - 1.2, sw - 1, sh - 1]
        net = Net(blobs)
        boxes, masks, scores = demo.im_detect(im, net)
        data = net.fed["data"]
        import zlib
        pr.update({"im_seed_shape_crc_" + tag: np.array([seed, H, W, zlib.crc32(im.tobytes())], np.int64),
                   "scale_" + tag: np.float64(scale), "im_info_" + tag: net.fed["im_info"],
                   "data_shape_" + tag: np.array(data.shape), "data_sum_" + tag: data.astype(np.float64).sum(),
                   "data_probe_" + tag: data[0, :, ::37, ::41].copy(),
                   "rois_" + tag: blobs["rois"].data, "rois_ext_" + tag: blobs["rois_ext"].data,
                   "mask_" + tag: blobs["mask_proposal"].data, "mask_ext_" + tag: blobs["mask_proposal_ext"].data,
                   "prob_" + tag: blobs["seg_cls_prob"].data, "prob_ext_" + tag: blobs["seg_cls_prob_ext"].data,
                   "out_boxes_" + tag: boxes, "out_masks_" + tag: masks, "out_scores_" + tag: scores})
        meta["tail_%s_boxes_dtype" % tag] = str(boxes.dtype)
    pr["cases"] = np.array([c[0] for c in pcases])
    save_parts(os.path.join(OUT, "ref_prep_tail.npz"), pr)

    # ---- recorded native calls (replayed on the GPU box through oracle/_ref) --------------------
    # `_nms` calls made by ProposalLayer.forward (the voting ones are in ref_voting.npz as keep lists;
    # the `_mv` calls are ref_voting.npz's cand_* inputs -> result_* outputs)
    rec = {}
    prop_calls = [c for c in native["nms"] if c[1] == cfg.TEST.RPN_NMS_THRESH]
    assert len(prop_calls) == len(cases)
    for (tag, *_), (dets, thr, keep) in zip(cases, prop_calls):
        rec.update({"dets_" + tag: dets, "thresh_" + tag: np.float64(thr), "keep_" + tag: keep.astype(np.int32)})
    rec["cases"] = np.array([c[0] for c in cases])
    np.savez_compressed(os.path.join(OUT, "ref_native_calls.npz"), **rec)

    meta["patched_files"] = _RefLoader.patched
    meta["numpy"] = np.__version__
    meta["native_calls"] = {"nms": len(native["nms"]), "mv": len(native["mv"])}
    import json
    with open(os.path.join(OUT, "ref_fixtures_meta.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
    print(json.dumps(meta, indent=1, sort_keys=True))
    for fn in sorted(os.listdir(OUT)):
        if fn.startswith("ref_"):
            print("%10d  %s" % (os.path.getsize(os.path.join(OUT, fn)), fn))


if __name__ == "__main__":
    main()
