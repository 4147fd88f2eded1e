"""The Kannala-Brandt camera model (camodocal::EquidistantCamera) beside the pinhole and MEI ones: the restatement against the reference's
compiled EquidistantCamera.cc (or its stored results) and its eigen-solver against LAPACK, then every library check of kb_camera_checks.py on
the emulation build (`not gpu`) and on libviwb.so (`gpu`)."""
import os
import subprocess

import pytest

import kb_camera_checks as kc
from viwb import lib as viwb_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    yield ctx
    ctx.close()


@pytest.fixture(scope="module")
def reference_kb():
    import viw_ref_kb as vrk
    if not vrk.available():
        pytest.skip("neither the compiled reference (oracle/_ref) nor its stored results (tests/golden/reference)")
    return vrk


def test_restatement_matches_reference_code(reference_kb):
    kc.check_restatement_vs_reference_code()


def test_eigenvalues_match_lapack():
    kc.check_eigenvalues_vs_lapack()


def test_kannala_brandt_tag_matches_the_header(tmp_path):
    prog = tmp_path / "tag.c"
    prog.write_text('#include <stdio.h>\n#include "viwb.h"\nint main(){printf("%zu %d\\n", sizeof(viwb_camera), (int)VIWB_CAMERA_KANNALA_BRANDT); return 0;}\n')
    exe = tmp_path / "tag"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(prog)])
    size, kb = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert size == 80 and kb == viwb_lib.CAMERA_KANNALA_BRANDT


CHECKS = ["undistort_velocity_camera", "kb_sessions", "kb_feedback", "kb_closed_loop", "kb_errors"]


@pytest.mark.parametrize("name", CHECKS)
def test_kb_camera_library(emu, name):
    getattr(kc, "check_" + name)(emu)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHECKS)
def test_gpu_kb_camera_library(gpu_ctx, name):
    getattr(kc, "check_" + name)(gpu_ctx)
