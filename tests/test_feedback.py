"""The estimator -> tracker feedback (viwb_predict_pts, viwb_tracker_feedback): the restatements against the reference's code (compiled, or its
stored results), then every check of feedback_checks.py on the emulation build (`not gpu`) and on libviwb.so (`gpu`)."""
import pytest

import feedback_checks as fc
from viwb import lib as viwb_lib


@pytest.fixture(scope="module")
def emu():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    yield ctx
    ctx.close()


@pytest.fixture(scope="module")
def reference_feedback():
    import viw_ref_feedback as vrf
    if not vrf.available():
        pytest.skip("neither the compiled reference (oracle/_ref) nor its stored results (tests/golden/reference)")
    return vrf


@pytest.mark.parametrize("cid", [1, 2, 3, 4])
def test_predict_restatement_matches_reference_code(reference_feedback, cid):
    fc.check_predict_restatement_vs_reference_code(cid)


def test_feedback_restatement_matches_reference_code(reference_feedback):
    fc.check_feedback_restatement_vs_reference_code()


@pytest.mark.parametrize("cid", [1, 2, 3, 4])
def test_predict_pts(emu, cid):
    fc.check_predict_pts(emu, cid)


def test_tracker_feedback(emu):
    fc.check_tracker_feedback(emu)


def test_fallback_rows_static_scene(emu):
    fc.check_fallback_rows_static_scene(emu)


def test_closed_loop(emu):
    fc.check_closed_loop(emu)


def test_unchanged_path(emu):
    fc.check_unchanged_path(emu)


def test_feedback_errors(emu):
    fc.check_feedback_errors(emu)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [1, 2, 3, 4])
def test_gpu_predict_pts(gpu_ctx, cid):
    fc.check_predict_pts(gpu_ctx, cid)


@pytest.mark.gpu
def test_gpu_tracker_feedback(gpu_ctx):
    fc.check_tracker_feedback(gpu_ctx)


@pytest.mark.gpu
def test_gpu_fallback_rows_static_scene(gpu_ctx):
    fc.check_fallback_rows_static_scene(gpu_ctx)


@pytest.mark.gpu
def test_gpu_closed_loop(gpu_ctx):
    fc.check_closed_loop(gpu_ctx)


@pytest.mark.gpu
def test_gpu_unchanged_path(gpu_ctx):
    fc.check_unchanged_path(gpu_ctx)


@pytest.mark.gpu
def test_gpu_feedback_errors(gpu_ctx):
    fc.check_feedback_errors(gpu_ctx)
