"""The MEI camera model (camodocal::CataCamera) beside the pinhole one: the restatements against the reference's compiled CataCamera.cc (or its
stored results), then every library check of camera_checks.py on the emulation build (`not gpu`) and on libviwb.so (`gpu`)."""
import ctypes as C
import os
import subprocess

import pytest

import camera_checks as cc
from viwb import lib as viwb_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    yield ctx
    ctx.close()


@pytest.fixture(scope="module")
def reference_camera():
    import viw_ref_camera as vrc
    if not vrc.available():
        pytest.skip("neither the compiled reference (oracle/_ref) nor its stored results (tests/golden/reference)")
    return vrc


def test_restatement_matches_reference_code(reference_camera):
    cc.check_restatement_vs_reference_code()


def test_feedback_restatement_matches_reference_code(reference_camera):
    cc.check_feedback_restatement_vs_reference_code()


def test_track_image_restatement_matches_reference_code():
    import viw_ref
    cv2 = pytest.importorskip("cv2")
    if not viw_ref.live():
        pytest.skip("the reference's FeatureTracker calls back into cv2 at every tick: it needs the compiled reference (VIWB_REFERENCE_DIR)")
    was = cv2.useOptimized(); cv2.setUseOptimized(False)             # goodFeaturesToTrack's scalar path is the specification
    try:
        cc.check_track_image_vs_reference_code(cv2)
    finally:
        cv2.setUseOptimized(was)


def test_camera_struct_size_matches_the_header(tmp_path):
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "viwb.h"\nint main(){printf("%zu %d %d\\n", sizeof(viwb_camera), (int)VIWB_CAMERA_PINHOLE, (int)VIWB_CAMERA_MEI); return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(prog)])
    size, pin, mei = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert size == C.sizeof(viwb_lib.Camera) and (pin, mei) == (viwb_lib.CAMERA_PINHOLE, viwb_lib.CAMERA_MEI)


CHECKS = ["undistort_velocity_camera", "mei_sessions", "mei_feedback", "mei_closed_loop", "pinhole_through_camera_entry", "camera_errors"]


@pytest.mark.parametrize("name", CHECKS)
def test_camera_library(emu, name):
    getattr(cc, "check_" + name)(emu)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHECKS)
def test_gpu_camera_library(gpu_ctx, name):
    getattr(cc, "check_" + name)(gpu_ctx)
