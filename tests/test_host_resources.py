"""Ownership of the library's CUDA resources (csrc/m3t_b200_owned.h): only the owner header creates or releases them,
nothing leaks, and a call refused because a resource could not be created leaves its context as it was
(m3tb_debug_resources injects the failure; nothing here allocates until memory runs out)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
OWNER_HEADER = "m3t_b200_owned.h"
RAW_CALLS = re.compile(r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|"
                       r"cudaEventDestroy)\s*\(")
I34 = np.eye(4, dtype=np.float32)[:3]
GEN = dict(n_divides=1, n_points=50, image_size=200)


def test_only_the_owner_header_creates_or_releases_resources():
    found = {}
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".h")):
            continue
        text = re.sub(r"//[^\n]*|/\*.*?\*/", "", open(os.path.join(CSRC, name)).read(), flags=re.S)
        calls = sorted(set(RAW_CALLS.findall(text)))
        if calls:
            found[name] = calls
    assert set(found) == {OWNER_HEADER}, found
    assert {"cudaMalloc", "cudaMallocHost", "cudaFree", "cudaFreeHost", "cudaStreamCreateWithFlags",
            "cudaStreamDestroy", "cudaEventCreateWithFlags", "cudaEventDestroy"} <= set(found[OWNER_HEADER])


# ---- GPU part ------------------------------------------------------------------------------------------------------

def _live(capi):
    return capi.debug_resources(-1)


def _params(capi, wl, n_bins=None, n_lines_max=None):
    rp, dp = capi.region_params(wl.region), capi.depth_params(wl.depth)
    if n_bins:
        rp.n_histogram_bins = n_bins
    if n_lines_max:
        rp.n_lines_max = n_lines_max
    return rp, dp, capi.OptimizerParams(wl.tikhonov_rotation, wl.tikhonov_translation)


def _rendering(synth, size, seed=0):
    img = np.random.default_rng(seed).integers(0, 65535, (size, size), dtype=np.uint16)
    return synth.Rendering(img, 10.0, 12.0, 1.0, 0.5, 0.25, 0, True)


def _pinned(a):
    import torch
    t = torch.empty(a.shape, dtype=getattr(torch, str(a.dtype)), pin_memory=True)
    t.numpy()[...] = a
    return t


def _step(ctx, wl):
    ctx.set_poses(wl.start_body2world)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    return ctx.get_poses()


class Scene:
    """Two tracked bodies (region + depth) in a context with every kind of object: models, a generated depth model
    (slot 1), pooled frames, body geometry, a rendered device renderer, an uploaded rendering, shared histograms and a
    kinematic structure, after one tracking step. Camera 2 is free for the uploads outside the pool."""

    def __init__(self, capi, synth):
        self.capi, self.synth = capi, synth
        self.wl = wl = synth.make_workload("c2", n_bodies=2, n_divides=2)
        self.gen = capi.model_params(**GEN)
        self.tri, self.diam = synth.prism_triangles()
        self.ico, self.ico_diam = synth.icosphere_triangles(n_divides=1)
        ci = wl.color_intrinsics
        self.small = type(ci)(*[getattr(ci, f) for f, _ in type(ci)._fields_])
        self.small.width, self.small.height = 320, 240
        self.small_frame = np.full((240, 320, 3), 90, np.uint8)
        self.pinned = [_pinned(self.small_frame), _pinned(wl.color_frames[:2]), _pinned(wl.depth_frames[:2])]

    def base(self):
        capi, synth, wl = self.capi, self.synth, self.wl
        ctx = capi.Context(0, max_bodies=2, max_cameras=3, max_models=2)
        ctx.set_region_model(0, wl.region_model)
        ctx.set_depth_model(0, wl.depth_model)
        for b in range(2):
            ctx.set_color_camera(b, wl.color_intrinsics, wl.color_world2camera)
            ctx.set_depth_camera(b, wl.depth_intrinsics, wl.depth_world2camera, wl.depth_scale)
        ctx.upload_color_batch(0, wl.color_frames[:2])
        ctx.upload_depth_batch(0, wl.depth_frames[:2])
        for b in range(2):
            ctx.set_body(b, *_params(capi, wl), 0, 0, b, b)
        for b in range(2):
            ctx.set_body_geometry(b, self.tri, I34, self.diam, True, b + 1, 7)
        ctx.generate_depth_model(1, 0, (), self.gen)
        ctx.set_focused_renderer(0, "color", 0, [0, 1], [0], image_size=64)
        ctx.render()
        ctx.upload_rendering(0, "depth_depth", _rendering(synth, 32))
        ctx.share_color_histograms(1, 0)
        ctx.set_structure(0, synth.StructureSpec(links=[synth.LinkSpec(body=1, parent=-1, body2joint=I34,
                                                                       joint2parent=I34)]))
        ctx.start_modalities(0)
        _step(ctx, wl)
        ctx.synchronize()
        return ctx

    def cases(self):
        """(name, prefix, call): `call` is an entry point that creates resources; `prefix` (or None) sets it up."""
        capi, synth, wl = self.capi, self.synth, self.wl
        rp32, dp, op = _params(capi, wl, n_bins=32)
        rp_long = _params(capi, wl, n_lines_max=2 * wl.region.n_lines_max)[0]
        bodyless = synth.StructureSpec(links=[synth.LinkSpec(body=-1, parent=-1, body2joint=I34, joint2parent=I34,
                                                             free_directions=(1, 0, 0, 0, 0, 0))])
        step = lambda c: c.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)  # noqa: E731
        camera2 = lambda c: c.set_color_camera(2, self.small, wl.color_world2camera)  # noqa: E731
        more_renderers = lambda c: [c.set_focused_renderer(r, "depth", 0, [0, 1], [0], image_size=16)  # noqa: E731
                                    for r in range(1, 8)]  # the render lists outgrow their first table
        pinned_frames = lambda c: (c.upload_color_batch(0, self.pinned[1].numpy()),  # noqa: E731
                                   c.upload_depth_batch(0, self.pinned[2].numpy()))
        return [
            ("set_region_model", None, lambda c: c.set_region_model(0, wl.region_model)),
            ("set_depth_model", None, lambda c: c.set_depth_model(1, wl.depth_model)),
            ("generate_depth_model", None, lambda c: c.generate_depth_model(1, 1, (0,), self.gen)),
            ("debug_render_model_view", None, lambda c: c.debug_render_model_view(0, 3, params=self.gen)),
            ("set_body_32_bins", None, lambda c: c.set_body(0, rp32, dp, op, 0, 0, 0, 0)),
            ("shared_histogram_tables", lambda c: (c.share_color_histograms(1, -1), c.share_color_histograms(1, 1)),
             lambda c: c.start_modalities(0)),
            ("structure_tables", lambda c: c.set_structure(1, bodyless), step),
            ("state_tables", lambda c: c.set_body(0, rp_long, dp, op, 0, 0, 0, 0), step),
            ("set_body_geometry", None, lambda c: c.set_body_geometry(1, self.ico, I34, self.ico_diam, True, 2, 7)),
            ("set_focused_renderer_resize", None,
             lambda c: c.set_focused_renderer(0, "color", 0, [0, 1], [0], image_size=128)),
            ("set_focused_renderer_new", None, lambda c: c.set_focused_renderer(1, "depth", 0, [0], [0], image_size=64)),
            ("render_tables", more_renderers, lambda c: c.render()),
            ("upload_rendering_resize", None, lambda c: c.upload_rendering(0, "depth_depth", _rendering(synth, 48))),
            ("prefetch_frames", pinned_frames, lambda c: c.prefetch_frames()),
            ("upload_pageable_outside_pool", camera2, lambda c: c.upload_color(2, self.small_frame)),
            ("upload_pinned_outside_pool", camera2, lambda c: c.upload_color(2, self.pinned[0].numpy())),
            ("set_viewer_new", None, lambda c: c.set_viewer(0, "color", 0, [0, 1])),
            ("update_viewers_tables", lambda c: c.set_viewer(0, "color", 0, [0, 1]), lambda c: c.update_viewers()),
            ("set_full_renderer_new", None, lambda c: c.set_full_renderer(0, "color", 0, [0, 1])),
            ("render_full_tables", lambda c: c.set_full_renderer(0, "color", 0, [0, 1]), lambda c: c.render_full()),
            ("generate_region_model", None, lambda c: c.generate_region_model(1, 0, (), self.gen)),
        ]

    def readbacks(self, ctx):
        m = ctx.get_depth_model(1)
        r = ctx.get_rendering(0)
        nb = self.wl.region.n_histogram_bins
        out = [m.orientations, m.view_scalars, m.points, r["depth"], r["silhouette"], r["visible"],
               np.float32([r[k] for k in ("corner_u", "corner_v", "scale", "projection_term_a", "projection_term_b")])]
        for b in range(2):
            out += list(ctx.get_histograms(b, nb))
        out += list(ctx.get_link_poses(0, 1))
        return [np.ascontiguousarray(a).view(np.uint8) for a in out]


def _run_leak_sequence():
    """Every entry point that creates resources, on one context; then the context is destroyed. Run in a process of
    its own, so that no other context is alive."""
    import importlib
    capi = importlib.import_module("3dobjecttracking_b200.capi")
    synth = importlib.import_module("3dobjecttracking_b200.synth")
    assert _live(capi) == 0
    k = 1
    while True:  # every failing creation of a context leaves nothing behind
        capi.debug_resources(k)
        try:
            ctx = capi.Context(0, 1, 1, 1)
        except capi.M3TBError:
            capi.debug_resources(0)
            assert _live(capi) == 0, k
            k += 1
            continue
        capi.debug_resources(0)
        ctx.close()
        break
    assert k > 5 and _live(capi) == 0
    s = Scene(capi, synth)
    ctx = s.base()
    ctx.set_region_model(0, s.wl.region_model)  # replacing a model
    for name, prefix, call in s.cases():
        if prefix:
            prefix(ctx)
        call(ctx)
        if name == "prefetch_frames":
            _step(ctx, s.wl)
    _step(ctx, s.wl)
    ctx.set_focused_renderer(0, "color", 0, [0, 1], [0], image_size=64)  # 64 -> 128 -> 64
    ctx.close()
    assert _live(capi) == 0
    print("leak sequence ok")


@pytest.mark.gpu
def test_nothing_leaks():
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_host_resources as t; t._run_leak_sequence()"
            % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "leak sequence ok" in r.stdout


@pytest.mark.gpu
def test_replacing_objects_does_not_leak(capi, synth):
    s = Scene(capi, synth)
    ctx = s.base()
    rp, dp, op = _params(capi, s.wl)
    rp32 = _params(capi, s.wl, n_bins=32)[0]

    def replace():
        ctx.set_region_model(0, s.wl.region_model)
        ctx.set_depth_model(1, s.wl.depth_model)
        ctx.generate_depth_model(1, 0, (), s.gen)
        for p in (rp32, rp):
            ctx.set_body(0, p, dp, op, 0, 0, 0, 0)
        for tri, diam in ((s.ico, s.ico_diam), (s.tri, s.diam)):
            ctx.set_body_geometry(1, tri, I34, diam, True, 2, 7)
        for size in (128, 64):
            ctx.set_focused_renderer(0, "color", 0, [0, 1], [0], image_size=size)
        for size in (48, 32):
            ctx.upload_rendering(0, "depth_depth", _rendering(synth, size))
        _step(ctx, s.wl)
        return _live(capi)

    first = replace()
    assert replace() == first
    ctx.close()


@pytest.mark.gpu
def test_a_failed_creation_changes_nothing(capi, synth):
    s = Scene(capi, synth)
    refused = {}
    for name, prefix, call in s.cases():
        twin = s.base()
        if prefix:
            prefix(twin)
        expect = _step(twin, s.wl)
        twin.close()
        k = 1
        while True:
            ctx = s.base()
            if prefix:
                prefix(ctx)
            before, live = s.readbacks(ctx), _live(capi)
            capi.debug_resources(k)
            try:
                call(ctx)
                failed = None
            except capi.M3TBError as e:
                failed = str(e)
            finally:
                capi.debug_resources(0)
            if failed is None:
                ctx.close()
                break
            assert failed.startswith("status -2:") and "out of memory" in failed and ".create(" in failed, \
                (name, k, failed)
            assert _live(capi) == live, (name, k)
            after = s.readbacks(ctx)
            assert all(np.array_equal(a, b) for a, b in zip(before, after)), (name, k)
            if name == "set_focused_renderer_new":  # no renderer 1 came into being
                with pytest.raises(capi.M3TBError, match="renderer not set"):
                    ctx.attach_renderer(0, "depth_depth", 1)
            got = _step(ctx, s.wl)
            assert np.array_equal(got.view(np.uint32), expect.view(np.uint32)), (name, k)
            ctx.close()
            k += 1
        refused[name] = k - 1
    print("refused creations per call:", refused)
    assert all(n > 0 for n in refused.values()), refused  # every call above has something to create
    assert refused["generate_depth_model"] >= 10 and refused["prefetch_frames"] >= 15, refused
