"""The resident FeatureManager's windows solved where they are (viwb_features_batch_create and the *_batch feedback calls): every check of
features_batch_checks.py on the emulation build (`not gpu`) and on libviwb.so (`gpu`), and one scripted sequence on the sanitizer build of the
emulation."""
import os
import subprocess
import sys

import pytest

import features_batch_checks as fbc
from viwb import lib as viwb_lib

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    yield ctx
    ctx.close()


def test_scripts(emu):
    fbc.check_scripts(emu)


def test_closed_loop(emu):
    fbc.check_closed_loop(emu)


def test_h2d_bytes(emu):
    fbc.check_h2d_bytes(emu)


def test_launches_do_not_depend_on_streams(emu):
    fbc.check_launches_do_not_depend_on_streams(emu)


def test_errors(emu):
    fbc.check_errors(emu)


def test_sanitized_script():
    """one stereo script of twin lists and the refusals on the ASan / UBSan build of the emulation, in a child process that preloads libasan"""
    from emu import build_emu
    built = build_emu.build_sanitized()
    if built is None:
        pytest.skip("the toolchain has no libasan")
    lib, asan = built
    root = os.path.dirname(HERE)
    code = ("import sys; sys.path[:0] = [%r, %r, %r]\n"
            "from viwb import lib; import features_batch_checks as fbc\n"
            "ctx = lib.Context(0, %r); fbc.run_twins(ctx, 2, 13, 10.0 / 460.0, 10); fbc.check_errors(ctx); ctx.close(); print('ok')\n"
            % (HERE, os.path.join(root, "viw-fusion_b200", "python"), os.path.join(root, "oracle"), lib))
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-4000:]


@pytest.mark.gpu
def test_gpu_scripts(gpu_ctx):
    fbc.check_scripts(gpu_ctx)


@pytest.mark.gpu
def test_gpu_closed_loop(gpu_ctx):
    fbc.check_closed_loop(gpu_ctx)


@pytest.mark.gpu
def test_gpu_h2d_bytes(gpu_ctx):
    fbc.check_h2d_bytes(gpu_ctx)


@pytest.mark.gpu
def test_gpu_launches_do_not_depend_on_streams(gpu_ctx):
    fbc.check_launches_do_not_depend_on_streams(gpu_ctx)


@pytest.mark.gpu
def test_gpu_errors(gpu_ctx):
    fbc.check_errors(gpu_ctx)
