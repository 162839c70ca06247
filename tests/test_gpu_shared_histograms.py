"""Shared ColorHistograms objects on the device (VERDICT r01 missing #3, second half): m3tb_share_color_histograms =
RegionModality::UseSharedColorHistograms (region_modality.cpp:168-179). k_histogram lets the members only add their line
pixels, k_histogram_shared initialises / updates the object once (tracker.cpp:435-443, 507-515) and hands every member
its copy of the histograms and of the lookup table. Bit-exact against the oracle's shared pass."""
import numpy as np
import pytest

from helpers import pose_error

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _workload(synth, n, bins):
    """c3 (region only, 32 bins) for 32 bins; c2 (200 lines + 200 points) at the given resolution otherwise."""
    wl = synth.make_workload("c2" if bins != 32 else "c3", n_bodies=n, n_lines=200, n_points=200 if bins != 32 else 0,
                             n_divides=3, seed=9)
    wl.region.n_histogram_bins = bins
    return wl


@pytest.mark.parametrize("bins", [2, 8, 16, 32, 64])
def test_shared_histograms_bit_exact(capi, oracle, synth, bins):
    n = 5
    wl = _workload(synth, n, bins)
    wl.histogram_owner = np.array([0, 0, 2, 2, -1], np.int32)
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.start_modalities(0)
    ctx.start_modalities(0)

    def check(stage):
        for b in range(n):
            hf, hb = ctx.get_histograms(b, bins)
            assert np.array_equal(_bits(hf), _bits(orc.hist_f[b])), (stage, b)
            assert np.array_equal(_bits(hb), _bits(orc.hist_b[b])), (stage, b)
        for a, b in ((0, 1), (2, 3)):
            ha, hb_ = ctx.get_histograms(a, bins), ctx.get_histograms(b, bins)
            assert np.array_equal(_bits(ha[0]), _bits(hb_[0])) and np.array_equal(_bits(ha[1]), _bits(hb_[1])), (stage, a, b)

    check("start")
    # the shared object differs from what the owner would have had alone
    alone = _workload(synth, n, bins)
    o2 = oracle.OracleTracker(alone, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    o2.start_modalities(0)
    assert np.abs(o2.hist_f[0] - orc.hist_f[0]).max() > 1e-6
    assert np.array_equal(_bits(o2.hist_f[4]), _bits(orc.hist_f[4]))
    for frame in range(2):
        # the lookup tables the tracking kernels read are the shared ones: same poses as the oracle after a step
        orc.tracking_step(frame)
        ctx.tracking_step(frame, wl.n_corr_iterations, wl.n_update_iterations)
        # 64-bin indices do not fit k_track2's u16 colour tile
        assert ctx.last_launch()["kernel"] == ("k_track" if bins > 32 else "k_track2"), ctx.last_launch()
        dt, dr = pose_error(ctx.get_poses(), orc.get_poses())
        assert np.median(dt) < 1e-5 and dt.max() < 5e-3, (frame, dt, dr)   # free-running (discrete events, DESIGN §5)
        ctx.set_poses(orc.get_poses())
        orc.calculate_results(frame)
        ctx.calculate_results(frame)
        check(f"frame {frame}")
    ctx.close()


def test_share_color_histograms_errors_and_release(capi, oracle, synth):
    wl = synth.make_workload("c2", n_bodies=3, n_lines=200, n_points=0, n_divides=2, seed=2)
    ctx = capi.context_from_workload(wl)
    ctx.share_color_histograms(1, 0)
    with pytest.raises(capi.M3TBError):
        ctx.share_color_histograms(2, 1)      # body 1 uses body 0's object: it cannot own one
    with pytest.raises(capi.M3TBError):
        ctx.share_color_histograms(0, -1)     # body 0 owns an object that body 1 still uses
    ctx.start_modalities(0)
    h0, h1 = ctx.get_histograms(0, 16), ctx.get_histograms(1, 16)
    assert np.array_equal(_bits(h0[0]), _bits(h1[0]))
    # set_histograms on a member sets the object for every user
    uni = np.full(16 ** 3, 1.0 / 16 ** 3, np.float32)
    ctx.set_histograms(1, uni, uni)
    assert np.array_equal(_bits(ctx.get_histograms(0, 16)[0]), _bits(uni))
    # release: both bodies private again -> the per-body result
    ctx.share_color_histograms(1, -1)
    ctx.share_color_histograms(0, -1)
    ctx.start_modalities(0)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.start_modalities(0)
    for b in range(3):
        hf, hb = ctx.get_histograms(b, 16)
        assert np.array_equal(_bits(hf), _bits(orc.hist_f[b])) and np.array_equal(_bits(hb), _bits(orc.hist_b[b])), b
    ctx.close()
