"""The full-renderer restatement (tests/full_renderer_reference.py) and the focused one (tests/render_reference.py) held
to the OpenGL images of the reference's renderer test (M3T/data/renderer_test/, checked by M3T/test/renderer_test.cpp
with CompareImages: a pixel is wrong when a channel differs by more than 1, and 10 wrong pixels are allowed). The
device renderers equal these restatements bit for bit (tests/test_gpu_full_renderers.py, tests/test_gpu_renderings.py),
so this pins them to an OpenGL driver."""
import numpy as np
import pytest

import full_renderer_reference as fr
import render_reference as rr

cv2 = pytest.importorskip("cv2")

MAX_WRONG = 10  # renderer_test.cpp: CompareToLoadedImage(..., 0, 10)
# The normal image of the dense schauma mesh (20,950 triangles) differs in 30 interior pixels. At each of them three or
# more sub-pixel triangles meet and a different one wins: the OpenGL driver snaps vertices to its sub-pixel grid, the
# restatement evaluates exact float edge functions. Coverage agrees everywhere (no pixel is background in one image and
# foreground in the other), which the test checks too.
NORMAL_WRONG = 30


@pytest.fixture(scope="module")
def scene():
    return fr.golden_scene()


@pytest.fixture(scope="module")
def full(scene):
    s = scene
    return fr.render_full(s.intrinsics, s.world2camera, s.poses, s.geometry, s.bodies, s.z_min, s.z_max, "body")


def test_full_depth_and_silhouette_meet_the_reference_rule(full):
    assert fr.wrong_pixels(full["silhouette"], fr.load_golden("silhouette_image.png")) == 0
    assert fr.wrong_pixels(full["depth"], fr.load_golden("depth_image.png")) <= MAX_WRONG


def test_full_images_are_not_flipped(full):
    for name, img in (("silhouette_image.png", full["silhouette"]), ("depth_image.png", full["depth"])):
        assert fr.wrong_pixels(img[::-1], fr.load_golden(name)) > 10000


def test_full_normal_image_differs_only_where_sub_pixel_triangles_meet(full):
    exp = fr.load_golden("normal_image.png")
    assert exp.shape == full["normal"].shape == (480, 640, 4)
    assert fr.wrong_pixels(full["normal"], exp) == NORMAL_WRONG
    assert np.array_equal(full["normal"][..., 3] == 0, exp[..., 3] == 0)
    # every wrong pixel is a schauma pixel (body_id 50)
    d = np.abs(full["normal"].astype(np.int64) - exp.astype(np.int64)).max(-1)
    assert (full["silhouette"][d > 1] == 50).all()


def test_focused_renderer_meets_the_reference_rule(scene):
    s = scene
    out = rr.render_focused(s.intrinsics, s.world2camera, s.poses, s.geometry, s.bodies, s.focused_referenced,
                            s.focused_size, s.z_min, s.z_max, "body")
    assert fr.wrong_pixels(out["silhouette"], fr.load_golden("focused_silhouette_image.png")) <= MAX_WRONG
    assert fr.wrong_pixels(out["depth"], fr.load_golden("focused_depth_image.png")) <= MAX_WRONG


def test_region_ids_and_z_range(scene):
    s = scene
    out = fr.render_full(s.intrinsics, s.world2camera, s.poses, s.geometry, s.bodies, 0.2, 1.5, "region")
    assert set(np.unique(out["silhouette"])) == {0, 150}
    assert ((out["depth"] != 65535) == (out["silhouette"] != 0)).all()
    # Depth(value) (renderer.cpp:431) maps the drawn values back into the z range
    z = fr.depth_of(out, out["depth"][out["depth"] != 65535])
    assert 0.2 < z.min() and z.max() < 1.5
