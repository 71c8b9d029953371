"""Device-side prep_im_for_blob + im_list_to_blob (lib/utils/blob.py:17-50): bit for bit against the
float32 model of the device's resize rule (tests/cv_resize.py), and within 1e-4 of cv2 (the
reference's own resize, whose bits depend on IPP and the CPU): golden fixtures made with cv2
(tests/golden/make_golden.py) and a live cv2 call."""
import os

import numpy as np
import pytest
import torch

from tests import cv_resize as C

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _run(im, scale):
    from mnc_b200 import ops
    t = torch.from_numpy(np.ascontiguousarray(im[None])).cuda()
    return ops.prep_images(t, scale)[0].cpu().numpy().transpose(1, 2, 0)


@pytest.mark.parametrize("name", ["up", "cap", "down"])
def test_prep_matches_cv2_golden(name):
    from mnc_b200 import ops
    g = np.load(os.path.join(GOLD, "prep.npz"))
    im, want = g["im_" + name], g["out_" + name]
    sc, tgt, mx = g["scale_" + name]
    assert ops.im_scale_for(im.shape, int(tgt), int(mx)) == sc
    got = _run(im, float(sc))
    assert got.shape == want.shape
    model = C.prep(im[None], float(sc), ops.PIXEL_MEANS)[0].transpose(1, 2, 0)
    assert np.array_equal(got, model)
    # fp32 bilinear on values of magnitude <= 255: agreement to a few ulp of 255
    assert np.abs(got - want).max() < 1e-4


def test_prep_voc_sized_image_and_identity_scale():
    from oracle import oracle as O
    rng = np.random.default_rng(5)
    im = rng.integers(0, 256, size=(375, 500, 3), dtype=np.uint8)
    want, sc = O.prep_im_for_blob(im)
    assert sc == 1.6
    got = _run(im, sc)
    assert got.shape == (600, 800, 3) and np.abs(got - want).max() < 1e-4
    from mnc_b200 import ops
    assert np.array_equal(got, C.prep(im[None], sc, ops.PIXEL_MEANS)[0].transpose(1, 2, 0))
    im2 = O.synthetic_image(0, 600, 1000)
    blob, info = O.prep_blob(im2)             # scale 1.0: pure mean subtraction + transpose
    got2 = _run(im2, 1.0)
    assert np.array_equal(got2.transpose(2, 0, 1)[None], blob)


def test_detector_on_raw_images_equals_blob_path():
    from oracle import oracle as O
    from mnc_b200 import weights as Wt
    from mnc_b200.api import Detector
    w = Wt.make_weights(Wt.TINY_ARCH)
    det = Detector(w, max_batch=2, height=600, width=1000)
    ims = np.stack([O.synthetic_image(i, 600, 1000) for i in range(2)])
    b1, m1, s1, v1, sc = det.im_detect_images(ims)
    b1, m1, s1 = b1.copy(), m1.copy(), s1.copy()
    blob = np.concatenate([O.prep_blob(im)[0] for im in ims])
    b2, m2, s2, v2 = det.im_detect_batch(blob)
    assert sc == 1.0
    assert np.array_equal(b1, b2) and np.array_equal(m1, m2) and np.array_equal(s1, s2)
