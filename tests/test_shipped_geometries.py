"""The LK tracker, the detector and the session tracker at the image sizes of the reference's shipped configurations and at the pyramid-depth
boundaries (geometry_checks.py): on the emulation build (`not gpu`, a thinned set of sizes) and on libviwb.so (`gpu`, every size), where the TMA
staging is also held bit for bit to the reflect-101 staging.  Run with -s to see the per-case agreement numbers."""
import numpy as np
import pytest

import geometry_checks as gc
from viwb import lib as viwb_lib

GEOMS = [pytest.param(w, h, lv, id="%dx%d" % (w, h)) for w, h, lv in gc.GEOMETRIES]
STRIDE_EMU = [pytest.param(w, h, id="%dx%d" % (w, h)) for w, h in [(1241, 376), (600, 600), (300, 85)]]
DETECT = [pytest.param(*g, id="%dx%d" % g[:2]) for g in gc.DETECTOR_GEOMETRIES]
BATCH = [pytest.param(w, h, id="%dx%d" % (w, h)) for w, h in [(1241, 376), (600, 600)]]
SESSIONS = [pytest.param(1241, 376, 2, 6, 200, 30, True, id="1241x376-stereo"),
            pytest.param(600, 600, 1, 6, 150, 30, False, id="600x600-mono"),
            pytest.param(300, 85, 1, 6, 60, 15, False, id="300x85-mono")]


@pytest.fixture(scope="module")
def emu():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    yield ctx
    ctx.close()


def test_belt_reaches_every_tile_offset():
    """the belt puts points at every residue mod 16 along each edge, at every level's distances, all inside the image"""
    for w, h, _ in gc.GEOMETRIES:
        b = gc.border_belt(w, h)
        assert (b[:, 0] >= 0).all() and (b[:, 0] <= w - 1).all() and (b[:, 1] >= 0).all() and (b[:, 1] <= h - 1).all(), (w, h)
        for edge in range(4):
            e = b[64 * edge: 64 * (edge + 1)]
            along = e[:, 1] if edge < 2 else e[:, 0]
            assert set(np.floor(along).astype(int) % 16) == set(range(16)) and set(along - np.floor(along)) == set(gc.FRACS), (w, h, edge)
        assert ((w - 1 - b[:, 0] > 10) & (w - 1 - b[:, 0] < 14)).sum() >= 3, (w, h)       # windows that cross the right edge while iterating


# ------------------------------------------------------------------------------------------------ emulation build
@pytest.mark.parametrize("w,h,levels", GEOMS)
def test_lk_vs_opencv(emu, w, h, levels):
    gc.check_lk_vs_opencv(emu, w, h, levels, "emulation")


@pytest.mark.parametrize("w,h,levels", GEOMS)
def test_track_checked(emu, w, h, levels):
    gc.check_track_checked_vs_reference(emu, w, h, "emulation")


@pytest.mark.parametrize("w,h", BATCH)
def test_lk_batch(emu, w, h):
    gc.check_lk_batch_vs_reference(emu, w, h, "emulation")


@pytest.mark.parametrize("w,h", STRIDE_EMU)
def test_strides(emu, w, h):
    gc.check_strides(emu, w, h, "emulation")


@pytest.mark.parametrize("w,h,max_cnt,min_dist", DETECT)
def test_detector(emu, w, h, max_cnt, min_dist):
    gc.check_detector_geometry(emu, w, h, max_cnt, min_dist, "emulation")


@pytest.mark.parametrize("w,h,streams,ticks,max_cnt,min_dist,stereo", SESSIONS)
def test_session(emu, w, h, streams, ticks, max_cnt, min_dist, stereo):
    gc.check_session(emu, w, h, "emulation", streams, ticks, max_cnt, min_dist, stereo)


# ------------------------------------------------------------------------------------------------ H100
@pytest.mark.gpu
@pytest.mark.parametrize("w,h,levels", GEOMS)
def test_gpu_lk_vs_opencv(gpu_ctx, w, h, levels):
    gc.check_lk_vs_opencv(gpu_ctx, w, h, levels, "gpu (TMA staging)")


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,levels", GEOMS)
def test_gpu_track_checked(gpu_ctx, w, h, levels):
    gc.check_track_checked_vs_reference(gpu_ctx, w, h, "gpu (TMA staging)")


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", BATCH)
def test_gpu_lk_batch(gpu_ctx, w, h):
    gc.check_lk_batch_vs_reference(gpu_ctx, w, h, "gpu (TMA staging)")


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,levels", GEOMS)
def test_gpu_tma_matches_reflect_staging(monkeypatch, w, h, levels):
    """VIWB_LK_NO_TMA is read when an LK batch is built (the single-call entry points cache theirs in the context): a fresh context per setting"""
    def make_ctx(no_tma):
        if no_tma:
            monkeypatch.setenv("VIWB_LK_NO_TMA", "1")
        else:
            monkeypatch.delenv("VIWB_LK_NO_TMA", raising=False)
        return viwb_lib.Context(0)
    gc.check_tma_matches_reflect(make_ctx, w, h)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,levels", GEOMS)
def test_gpu_strides(gpu_ctx, w, h, levels):
    gc.check_strides(gpu_ctx, w, h, "gpu (TMA staging)")


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,max_cnt,min_dist", DETECT)
def test_gpu_detector(gpu_ctx, w, h, max_cnt, min_dist):
    gc.check_detector_geometry(gpu_ctx, w, h, max_cnt, min_dist, "gpu")


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,streams,ticks,max_cnt,min_dist,stereo", SESSIONS)
def test_gpu_session(gpu_ctx, w, h, streams, ticks, max_cnt, min_dist, stereo):
    gc.check_session(gpu_ctx, w, h, "gpu (TMA staging)", streams, ticks, max_cnt, min_dist, stereo)
