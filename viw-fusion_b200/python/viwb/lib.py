"""ctypes binding of libviwb.so (viw-fusion_b200/csrc), the CUDA implementation behind include/viwb.h.

No fallback of any kind: if the shared library is missing, or no CUDA device is usable, creating a Context raises.
`Context(device, libpath=...)` lets the CPU test-suite point the same binding at the test-only kernel-logic
emulation build (tests/emu/libviwb_emu.so); the product never does.
"""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.normpath(os.path.join(_HERE, "..", "..", "csrc", "libviwb.so"))

EXPORTS = ["viwb_create", "viwb_destroy", "viwb_last_error", "viwb_set_stream", "viwb_launch_count", "viwb_h2d_bytes", "viwb_set_profiling", "viwb_profile_count", "viwb_profile_get", "viwb_default_options",
           "viwb_default_globals", "viwb_factor_evaluate", "viwb_prior_evaluate", "viwb_window_solve", "viwb_gauge_reanchor",
           "viwb_marginalize", "viwb_optimization", "viwb_optimization_batch", "viwb_batch_create", "viwb_batch_reset_states",
           "viwb_batch_run", "viwb_batch_download", "viwb_batch_algorithmic_bytes", "viwb_batch_solve_launch", "viwb_batch_destroy",
           "viwb_debug_normal_equations", "viwb_lk_track", "viwb_track_checked", "viwb_lk_batch_create", "viwb_lk_batch_destroy",
           "viwb_lk_batch_upload", "viwb_lk_batch_run", "viwb_lk_batch_download", "viwb_lk_batch_algorithmic_bytes", "viwb_host_register",
           "viwb_host_unregister", "viwb_imu_preintegrate", "viwb_wheel_preintegrate", "viwb_outlier_rejection", "viwb_batch_outliers", "viwb_triangulate", "viwb_shift_depth", "viwb_predict_pts", "viwb_undistort_velocity", "viwb_undistort_velocity_camera",
           "viwb_set_mask", "viwb_good_features_to_track", "viwb_detector_create", "viwb_detector_destroy", "viwb_detector_detect", "viwb_detector_algorithmic_bytes",
           "viwb_tracker_create", "viwb_tracker_create_camera", "viwb_tracker_destroy", "viwb_tracker_track", "viwb_tracker_feedback", "viwb_tracker_download", "viwb_tracker_algorithmic_bytes",
           "viwb_solve_gyroscope_bias", "viwb_linear_alignment",
           "viwb_features_create", "viwb_features_destroy", "viwb_features_add", "viwb_features_add_tracked", "viwb_features_decisions", "viwb_features_triangulate",
           "viwb_features_window", "viwb_features_set_depth", "viwb_features_remove_outliers", "viwb_features_predict", "viwb_features_slide",
           "viwb_features_remove_failures", "viwb_features_download", "viwb_features_batch_create", "viwb_features_set_depth_batch",
           "viwb_features_remove_outliers_batch", "viwb_features_predict_batch"]


class ViwbError(RuntimeError):
    pass


def load(libpath=None):
    path = libpath or DEFAULT_LIB
    if not os.path.exists(path):
        raise ViwbError("libviwb.so not found at %s -- build it with __graft_entry__.build() (nvcc, sm_90a)" % path)
    lib = C.CDLL(path)
    lib.viwb_last_error.restype = C.c_char_p
    lib.viwb_launch_count.restype = C.c_longlong
    lib.viwb_h2d_bytes.restype = C.c_longlong
    lib.viwb_batch_algorithmic_bytes.restype = C.c_double
    lib.viwb_lk_batch_algorithmic_bytes.restype = C.c_double
    lib.viwb_lk_batch_algorithmic_bytes.argtypes = [C.c_void_p]
    lib.viwb_detector_algorithmic_bytes.restype = C.c_double
    lib.viwb_detector_algorithmic_bytes.argtypes = [C.c_void_p]
    lib.viwb_detector_destroy.argtypes = [C.c_void_p]
    lib.viwb_lk_batch_destroy.argtypes = [C.c_void_p]
    lib.viwb_lk_batch_destroy.restype = None
    lib.viwb_tracker_algorithmic_bytes.restype = C.c_double
    lib.viwb_tracker_algorithmic_bytes.argtypes = [C.c_void_p]
    lib.viwb_tracker_destroy.argtypes = [C.c_void_p]
    lib.viwb_tracker_destroy.restype = None
    lib.viwb_features_destroy.argtypes = [C.c_void_p]
    lib.viwb_features_destroy.restype = None
    return lib


def _dp(a):
    return a.ctypes.data_as(abi.c_double_p)


class Context:
    def __init__(self, device=0, libpath=None):
        self.lib = load(libpath)
        self.h = C.c_void_p()
        rc = self.lib.viwb_create(C.c_int(device), C.byref(self.h))
        if rc:
            raise ViwbError("viwb_create(device=%d) failed with %d: no usable CUDA device (there is no CPU fallback)" % (device, rc))

    def close(self):
        if self.h:
            self.lib.viwb_destroy(self.h)
            self.h = C.c_void_p()

    def _ck(self, rc, what):
        if rc:
            raise ViwbError("%s failed with %d: %s" % (what, rc, self.lib.viwb_last_error(self.h).decode()))

    def set_stream(self, cuda_stream_ptr):
        self._ck(self.lib.viwb_set_stream(self.h, C.c_void_p(cuda_stream_ptr)), "viwb_set_stream")

    def launch_count(self):
        return int(self.lib.viwb_launch_count(self.h))

    def h2d_bytes(self):
        return int(self.lib.viwb_h2d_bytes(self.h))

    def set_profiling(self, on):
        self._ck(self.lib.viwb_set_profiling(self.h, C.c_int(1 if on else 0)), "viwb_set_profiling")

    def profile(self):
        """{kernel name: (total ms, launches)} accumulated since set_profiling(True)."""
        out = {}
        for i in range(self.lib.viwb_profile_count(self.h)):
            name = C.create_string_buffer(64)
            ms, cnt = C.c_double(), C.c_longlong()
            self.lib.viwb_profile_get(self.h, C.c_int(i), name, C.c_int(64), C.byref(ms), C.byref(cnt))
            out[name.value.decode()] = (ms.value, cnt.value)
        return out

    # ---------------------------------------------------------------- factor level
    def factor_evaluate(self, ftype, globals_, consts, params, want_jac=True, null_jac=()):
        sizes = abi.FACTOR_BLOCK_SIZES[ftype]
        nres = abi.FACTOR_RESIDUALS[ftype]
        P = [np.ascontiguousarray(p, np.float64) for p in params]
        pp = (abi.c_double_p * len(P))(*[_dp(p) for p in P])
        res = np.zeros(nres)
        cst = np.ascontiguousarray(consts, np.float64) if consts is not None else None
        jacs = [None if (not want_jac or i in null_jac) else np.zeros((nres, s)) for i, s in enumerate(sizes)]
        jp = (abi.c_double_p * len(P))(*[(_dp(j) if j is not None else None) for j in jacs]) if want_jac else None
        self._ck(self.lib.viwb_factor_evaluate(self.h, C.c_int(ftype), C.byref(globals_), _dp(cst) if cst is not None else None, pp, _dp(res), jp),
                 "viwb_factor_evaluate")
        return res, jacs

    def prior_evaluate(self, prior, state, want_jac=True):
        st = np.ascontiguousarray(state[:abi.STATE_FIXED], np.float64)
        res = np.zeros(prior.n)
        jac = np.zeros((prior.n, abi.STATE_FIXED)) if want_jac else None
        self._ck(self.lib.viwb_prior_evaluate(self.h, C.byref(prior.c), _dp(st), _dp(res), _dp(jac) if want_jac else None), "viwb_prior_evaluate")
        return res, jac

    # ---------------------------------------------------------------- window level
    def window_solve(self, problem, state, options=None):
        st = np.array(state, np.float64, copy=True)
        opt = options if options is not None else abi.default_options()
        summ = abi.Summary()
        self._ck(self.lib.viwb_window_solve(self.h, C.byref(problem.c), _dp(st), C.byref(opt), C.byref(summ)), "viwb_window_solve")
        return st, summ

    def gauge_reanchor(self, problem, state_before, state):
        sb = np.ascontiguousarray(state_before, np.float64)
        st = np.array(state, np.float64, copy=True)
        self._ck(self.lib.viwb_gauge_reanchor(self.h, C.byref(problem.c), _dp(sb), _dp(st)), "viwb_gauge_reanchor")
        return st

    def marginalize(self, problem, state, flag):
        st = np.ascontiguousarray(state, np.float64)
        out = abi.PriorData()
        self._ck(self.lib.viwb_marginalize(self.h, C.byref(problem.c), _dp(st), C.c_int(flag), C.byref(out.c)), "viwb_marginalize")
        return out

    def optimization(self, problem, state, flag, options=None, want_prior=True):
        st = np.array(state, np.float64, copy=True)
        opt = options if options is not None else abi.default_options()
        summ = abi.Summary()
        out = abi.PriorData() if want_prior else None
        self._ck(self.lib.viwb_optimization(self.h, C.byref(problem.c), _dp(st), C.byref(opt), C.c_int(flag), C.byref(summ),
                                            C.byref(out.c) if out else None), "viwb_optimization")
        return st, summ, out

    def normal_equations(self, problem, state):
        st = np.ascontiguousarray(state, np.float64)
        T = abi.TANGENT_FIXED
        H, g = np.zeros((T, T)), np.zeros(T)
        lm = np.zeros((max(problem.num_landmarks, 1), 82))
        c = C.c_double()
        self._ck(self.lib.viwb_debug_normal_equations(self.h, C.byref(problem.c), _dp(st), _dp(H), _dp(g), _dp(lm), C.byref(c)),
                 "viwb_debug_normal_equations")
        return H, g, lm[: problem.num_landmarks], c.value

    def batch(self, problems, states, flags=None, options=None):
        return Batch(self, problems, states, flags, options)

    def optimization_batch(self, problems, states, flags, options=None, want_priors=True):
        """Host buffers in, host buffers out (the e2e path)."""
        B = len(problems)
        arr = (abi.Problem * B)()
        for i, p in enumerate(problems):
            p.fill(arr[i])
        sts = [np.array(s, np.float64, copy=True) for s in states]
        sp = (abi.c_double_p * B)(*[_dp(s) for s in sts])
        fl = (C.c_int32 * B)(*[int(f) for f in flags])
        opt = options if options is not None else abi.default_options()
        summ = (abi.Summary * B)()
        pri = [abi.PriorData() for _ in range(B)] if want_priors else None
        parr = None
        if want_priors:
            parr = (abi.Prior * B)()
            for i, p in enumerate(pri):
                parr[i] = p.c
        self._ck(self.lib.viwb_optimization_batch(self.h, C.c_int(B), arr, sp, C.byref(opt), fl, summ, parr), "viwb_optimization_batch")
        if want_priors:
            for i, p in enumerate(pri):
                p.c.valid, p.c.n, p.c.num_blocks = parr[i].valid, parr[i].n, parr[i].num_blocks
                for k in range(abi.NUM_FIXED_BLOCKS):
                    p.c.block_id[k], p.c.block_idx[k] = parr[i].block_id[k], parr[i].block_idx[k]
        return sts, list(summ), pri

    def prepare_optimization_batch(self, problems, states, flags, options=None):
        """Marshal the arguments of viwb_optimization_batch once; the returned callable is exactly one C-ABI call
        (host buffers in, host buffers out).  A C++ caller has no marshalling at all -- this keeps Python's out of timings."""
        B = len(problems)
        arr = (abi.Problem * B)()
        for i, p in enumerate(problems):
            p.fill(arr[i])
        src = [np.ascontiguousarray(s, np.float64) for s in states]
        sts = [s.copy() for s in src]
        sp = (abi.c_double_p * B)(*[_dp(s) for s in sts])
        fl = (C.c_int32 * B)(*[int(f) for f in flags])
        opt = options if options is not None else abi.default_options()
        summ = (abi.Summary * B)()
        pri = [abi.PriorData() for _ in range(B)]
        parr = (abi.Prior * B)()
        for i, p in enumerate(pri):
            parr[i] = p.c
        keep = (arr, src, sts, sp, fl, opt, summ, pri, parr, problems)

        def call():
            for s, d in zip(src, sts):      # the call updates the states in place: restore the inputs
                d[:] = s
            self._ck(self.lib.viwb_optimization_batch(self.h, C.c_int(B), arr, sp, C.byref(opt), fl, summ, parr), "viwb_optimization_batch")
            return sts, summ, parr
        call.keep = keep
        return call

    # ---------------------------------------------------------------- feature tracker
    def lk_track(self, prev_img, next_img, prev_pts, next_pts=None, max_level=3, max_iter=30, eps=0.01, flags=0, min_eig=1e-4):
        a = np.ascontiguousarray(prev_img, np.uint8)
        b = np.ascontiguousarray(next_img, np.uint8)
        h, w = a.shape
        p0 = np.ascontiguousarray(prev_pts, np.float32).reshape(-1, 2)
        n = len(p0)
        p1 = np.array(next_pts if next_pts is not None else p0, np.float32, copy=True).reshape(-1, 2)
        st = np.zeros(n, np.uint8)
        err = np.zeros(n, np.float32)
        self._ck(self.lib.viwb_lk_track(self.h, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), C.c_int(w), C.c_int(h), C.c_int(a.strides[0]),
                                        p0.ctypes.data_as(C.c_void_p), p1.ctypes.data_as(C.c_void_p), C.c_int(n), C.c_int(21), C.c_int(max_level),
                                        C.c_int(max_iter), C.c_float(eps), C.c_int(flags), C.c_float(min_eig), st.ctypes.data_as(C.c_void_p),
                                        err.ctypes.data_as(C.c_void_p)), "viwb_lk_track")
        return p1, st, err

    def track_checked(self, img_a, img_b, pts_a, mode=0, flow_back=True):
        a = np.ascontiguousarray(img_a, np.uint8)
        b = np.ascontiguousarray(img_b, np.uint8)
        h, w = a.shape
        p0 = np.ascontiguousarray(pts_a, np.float32).reshape(-1, 2)
        n = len(p0)
        p1 = np.zeros_like(p0)
        st = np.zeros(n, np.uint8)
        self._ck(self.lib.viwb_track_checked(self.h, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), C.c_int(w), C.c_int(h), C.c_int(a.strides[0]),
                                             p0.ctypes.data_as(C.c_void_p), p1.ctypes.data_as(C.c_void_p), C.c_int(n), C.c_int(mode),
                                             C.c_int(1 if flow_back else 0), st.ctypes.data_as(C.c_void_p)), "viwb_track_checked")
        return p1, st

    def outlier_rejection(self, problem, state, focal=460.0, thresh=3.0):
        st = np.ascontiguousarray(state, np.float64)
        out = np.zeros(max(problem.num_landmarks, 1), np.uint8)
        self._ck(self.lib.viwb_outlier_rejection(self.h, C.byref(problem.c), _dp(st), C.c_double(focal), C.c_double(thresh), out.ctypes.data_as(C.c_void_p)),
                 "viwb_outlier_rejection")
        return out[: problem.num_landmarks]

    def undistort_velocity(self, cam, pts, prev_un=None, has_prev=None, dt=0.05, want_velocity=True):
        """cam = (fx, fy, cx, cy, k1, k2, p1, p2) (viwb_undistort_velocity) or a Camera of either model (viwb_undistort_velocity_camera);
        pts float32 (n, 2) pixels -> (normalised points, velocities) as float32"""
        p = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
        n = len(p)
        un, vel = np.zeros((n, 2), np.float32), np.zeros((n, 2), np.float32)
        pv = None if prev_un is None else np.ascontiguousarray(prev_un, np.float32)
        hp = None if has_prev is None else np.ascontiguousarray(has_prev, np.uint8)
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        if isinstance(cam, Camera):
            fn, name, c = self.lib.viwb_undistort_velocity_camera, "viwb_undistort_velocity_camera", C.byref(cam)
        else:
            fn, name, c = self.lib.viwb_undistort_velocity, "viwb_undistort_velocity", (C.c_double * 8)(*[float(v) for v in cam])
        self._ck(fn(self.h, c, C.c_int(n), vp(p), vp(pv), vp(hp), C.c_double(dt), vp(un), vp(vel) if want_velocity else None), name)
        return un, vel

    def triangulate(self, state, stereo, frame, pt0, pt1, init_depth=5.0):
        st = np.ascontiguousarray(state, np.float64)
        s_, f_ = np.ascontiguousarray(stereo, np.int32), np.ascontiguousarray(frame, np.int32)
        a, b = np.ascontiguousarray(pt0, np.float64), np.ascontiguousarray(pt1, np.float64)
        out = np.zeros(len(s_))
        vp = lambda x: x.ctypes.data_as(C.c_void_p)
        self._ck(self.lib.viwb_triangulate(self.h, _dp(st), C.c_int(len(s_)), vp(s_), vp(f_), _dp(a), _dp(b), C.c_double(init_depth), _dp(out)), "viwb_triangulate")
        return out

    def shift_depth(self, uv, depth, marg_R, marg_P, new_R, new_P, init_depth=5.0):
        uv, depth = np.ascontiguousarray(uv, np.float64), np.ascontiguousarray(depth, np.float64)
        m = [np.ascontiguousarray(x, np.float64) for x in (marg_R, marg_P, new_R, new_P)]
        out = np.zeros(len(depth))
        self._ck(self.lib.viwb_shift_depth(self.h, C.c_int(len(depth)), _dp(uv), _dp(depth), _dp(m[0]), _dp(m[1]), _dp(m[2]), _dp(m[3]), C.c_double(init_depth), _dp(out)),
                 "viwb_shift_depth")
        return out

    def predict_pts(self, state, frame_count, start_frame, num_obs, pt0, depth):
        """Estimator::predictPtsInNextFrame over the caller's feature list -> (pts_cam [n, 3], valid [n] uint8)"""
        st = np.ascontiguousarray(state, np.float64)
        sf, no = np.ascontiguousarray(start_frame, np.int32), np.ascontiguousarray(num_obs, np.int32)
        p0, dep = np.ascontiguousarray(pt0, np.float64).reshape(-1, 3), np.ascontiguousarray(depth, np.float64)
        n = len(sf)
        assert len(no) == n and len(p0) == n and len(dep) == n
        out, valid = np.zeros((n, 3)), np.zeros(n, np.uint8)
        vp = lambda x: x.ctypes.data_as(C.c_void_p)
        self._ck(self.lib.viwb_predict_pts(self.h, _dp(st), C.c_int(frame_count), C.c_int(n), vp(sf), vp(no), _dp(p0), _dp(dep), _dp(out), vp(valid)), "viwb_predict_pts")
        return out, valid

    # ---------------------------------------------------------------- pre-integration (SURVEY 8 f-2)
    @staticmethod
    def _pack_intervals(dts, a_list, b_list):
        counts = np.array([len(d) for d in dts], np.int32)
        dt = np.ascontiguousarray(np.concatenate([np.asarray(d, np.float64) for d in dts]) if len(dts) else np.zeros(0))
        a = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float64).reshape(-1, 3) for x in a_list]) if len(a_list) else np.zeros((0, 3)))
        b = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float64).reshape(-1, 3) for x in b_list]) if len(b_list) else np.zeros((0, 3)))
        assert len(a) == len(dt) + len(dts) and len(b) == len(a)
        return counts, dt, a, b

    def imu_preintegrate(self, dts, accs, gyrs, ba, bg, noise):
        """n intervals: dts[i] (k_i,), accs[i] / gyrs[i] (k_i + 1, 3), ba / bg (n, 3), noise = (ACC_N, GYR_N, ACC_W, GYR_W) -> records (n, 287)"""
        counts, dt, a, g = self._pack_intervals(dts, accs, gyrs)
        n = len(counts)
        ba = np.ascontiguousarray(ba, np.float64).reshape(n, 3); bg = np.ascontiguousarray(bg, np.float64).reshape(n, 3)
        nz = np.ascontiguousarray(noise, np.float64)
        rec = np.zeros((n, abi.IMU_DOUBLES))
        vp = lambda x: x.ctypes.data_as(C.c_void_p)
        self._ck(self.lib.viwb_imu_preintegrate(self.h, C.c_int(n), vp(counts), vp(dt), vp(a), vp(g), vp(ba), vp(bg), vp(nz), vp(rec)), "viwb_imu_preintegrate")
        return rec

    def wheel_preintegrate(self, dts, vels, gyrs, s, td, noise):
        """n intervals: vels[i] / gyrs[i] (k_i + 1, 3), s (n, 3) = sx, sy, sw, td (n,), noise = (VEL_N_wheel, GYR_N_wheel) -> records (n, 78)"""
        counts, dt, v, g = self._pack_intervals(dts, vels, gyrs)
        n = len(counts)
        s = np.ascontiguousarray(s, np.float64).reshape(n, 3); td = np.ascontiguousarray(td, np.float64).reshape(n)
        nz = np.ascontiguousarray(noise, np.float64)
        rec = np.zeros((n, abi.WHEEL_DOUBLES))
        vp = lambda x: x.ctypes.data_as(C.c_void_p)
        self._ck(self.lib.viwb_wheel_preintegrate(self.h, C.c_int(n), vp(counts), vp(dt), vp(v), vp(g), vp(s), vp(td), vp(nz), vp(rec)), "viwb_wheel_preintegrate")
        return rec

    def solve_gyroscope_bias(self, R, imu_records):
        """solveGyroscopeBias (initial/initial_aligment.cpp:14-37): R (F, 3, 3), imu_records (F - 1, 287) -> delta_bg (3,)"""
        R = np.ascontiguousarray(R, np.float64); rec = np.ascontiguousarray(imu_records, np.float64)
        out = np.zeros(3)
        vp = lambda x: x.ctypes.data_as(C.c_void_p)
        self._ck(self.lib.viwb_solve_gyroscope_bias(self.h, C.c_int(len(R)), vp(R), vp(rec), vp(out)), "viwb_solve_gyroscope_bias")
        return out

    def linear_alignment(self, R, T, imu_records, wheel_records, tic, rio, tio, g_norm):
        """LinearAlignment[WithWheel] + RefineGravity[WithWheel] (:66-334); wheel_records None = camera + IMU only -> (aligned, g, x)"""
        F = len(R)
        R = np.ascontiguousarray(R, np.float64); T = np.ascontiguousarray(T, np.float64); rec = np.ascontiguousarray(imu_records, np.float64)
        w = np.ascontiguousarray(wheel_records, np.float64) if wheel_records is not None else None
        tic = np.ascontiguousarray(tic, np.float64)
        rio = np.ascontiguousarray(rio, np.float64) if rio is not None else None
        tio = np.ascontiguousarray(tio, np.float64) if tio is not None else None
        g, x, xs, ok = np.zeros(3), np.zeros(3 * F + 4), C.c_int32(0), C.c_int32(0)
        vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
        self._ck(self.lib.viwb_linear_alignment(self.h, C.c_int(F), vp(R), vp(T), vp(rec), vp(w), vp(tic), vp(rio), vp(tio), C.c_double(g_norm), vp(g), vp(x),
                                                C.byref(xs), C.byref(ok)), "viwb_linear_alignment")
        return bool(ok.value), g, x[: xs.value].copy()

    def visual_imu_alignment(self, R, T, dts, accs, gyrs, noise, bg0, wheel_records, tic, rio, tio, g_norm):
        """VisualIMUAlignment (:336-344) as the reference sequences it: gyroscope bias from the current pre-integrations, repropagation of every
        interval with ba = 0, bg = bg0 + delta_bg (viwb_imu_preintegrate on the same buffers), linear alignment.  All three steps on the device."""
        n = len(dts)
        rec0 = self.imu_preintegrate(dts, accs, gyrs, np.zeros((n, 3)), np.tile(np.asarray(bg0, np.float64), (n, 1)), noise)
        dbg = self.solve_gyroscope_bias(R, rec0)
        rec = self.imu_preintegrate(dts, accs, gyrs, np.zeros((n, 3)), np.tile(np.asarray(bg0, np.float64) + dbg, (n, 1)), noise)
        ok, g, x = self.linear_alignment(R, T, rec, wheel_records, tic, rio, tio, g_norm)
        return {"ok": ok, "delta_bg": dbg, "imu": rec, "g": g, "x": x}

    def set_mask(self, width, height, pts, track_cnt, min_dist, base_mask=None, want_mask=True):
        """FeatureTracker::setMask(): returns (mask uint8 [height, width] or None, surviving indices in visiting order)"""
        p = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
        c = np.ascontiguousarray(track_cnt, np.int32)
        n = len(p)
        keep, nk = np.zeros(max(n, 1), np.int32), C.c_int(0)
        mask = np.zeros((height, width), np.uint8) if want_mask else None
        bm = None if base_mask is None else np.ascontiguousarray(base_mask, np.uint8)
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        self._ck(self.lib.viwb_set_mask(self.h, C.c_int(width), C.c_int(height), vp(p), vp(c), C.c_int(n), C.c_int(int(min_dist)), vp(bm), vp(mask), vp(keep), C.byref(nk)),
                 "viwb_set_mask")
        return mask, keep[: nk.value].copy()

    def good_features_to_track(self, img, max_corners, quality, min_dist, mask=None, capacity=None):
        """cv2.goodFeaturesToTrack(img, max_corners, quality, min_dist, mask=mask) -> float32 (n, 2)"""
        assert img.dtype == np.uint8 and img.ndim == 2 and img.strides[1] == 1
        h, w = img.shape
        cap = capacity or (max_corners if max_corners > 0 else 1024)
        out, n = np.zeros((cap, 2), np.float32), C.c_int(0)
        m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        self._ck(self.lib.viwb_good_features_to_track(self.h, vp(img), C.c_int(w), C.c_int(h), C.c_int(img.strides[0]), C.c_int(max_corners), C.c_double(quality),
                                                      C.c_double(min_dist), vp(m), C.c_int(w), vp(out), C.c_int(cap), C.byref(n)), "viwb_good_features_to_track")
        return out[: n.value].copy()

    def detector(self, streams, width, height, max_pts, min_dist):
        return Detector(self, streams, width, height, max_pts, min_dist)

    def lk_batch(self, streams, width, height, max_points, stereo=True, flow_back=True):
        return LkBatch(self, streams, width, height, max_points, stereo, flow_back)

    def tracker(self, streams, width, height, cam0, cam1=None, max_cnt=150, min_dist=30, flow_back=True):
        return Tracker(self, streams, width, height, cam0, cam1, max_cnt, min_dist, flow_back)

    def features(self, streams, max_rows, stereo, min_parallax, focal_length=460.0, init_depth=5.0, max_features=0):
        return Features(self, streams, max_rows, stereo, min_parallax, focal_length, init_depth, max_features)

    def host_register(self, arr):
        self._ck(self.lib.viwb_host_register(self.h, C.c_void_p(arr.ctypes.data), C.c_size_t(arr.nbytes)), "viwb_host_register")

    def host_unregister(self, arr):
        self._ck(self.lib.viwb_host_unregister(self.h, C.c_void_p(arr.ctypes.data)), "viwb_host_unregister")


CAMERA_PINHOLE, CAMERA_MEI, CAMERA_KANNALA_BRANDT = 0, 1, 2
MAX_LANDMARKS = 1000          # VIWB_MAX_LANDMARKS, the per-stream landmark stride of the viwb_features_* arrays


class Camera(C.Structure):
    """viwb_camera: a camera of any model (include/viwb.h).  Build one with Camera.pinhole(...), Camera.mei(...) or Camera.kannala_brandt(...)."""
    _fields_ = [("model", C.c_int32), ("p", C.c_double * 9)]

    @classmethod
    def pinhole(cls, fx, fy, cx, cy, k1, k2, p1, p2):
        return cls(CAMERA_PINHOLE, (C.c_double * 9)(fx, fy, cx, cy, k1, k2, p1, p2, 0.0))

    @classmethod
    def mei(cls, xi, k1, k2, p1, p2, gamma1, gamma2, u0, v0):
        """the parameters in the order of a camodocal MEI yaml file (CataCamera's constructor)"""
        return cls(CAMERA_MEI, (C.c_double * 9)(xi, k1, k2, p1, p2, gamma1, gamma2, u0, v0))

    @classmethod
    def kannala_brandt(cls, k2, k3, k4, k5, mu, mv, u0, v0):
        """the parameters in the order of a camodocal KANNALA_BRANDT yaml file (EquidistantCamera::Parameters); Kalibr's `equidistant`
        intrinsics (fu, fv, pu, pv) and distortion (k1..k4) are mu, mv, u0, v0 and k2..k5"""
        return cls(CAMERA_KANNALA_BRANDT, (C.c_double * 9)(k2, k3, k4, k5, mu, mv, u0, v0, 0.0))


class TrackerConfig(C.Structure):
    _fields_ = [("max_cnt", C.c_int), ("min_dist", C.c_int), ("flow_back", C.c_int), ("stereo", C.c_int), ("cam", C.c_double * 16)]


class Tracker:
    """`streams` FeatureTracker sessions resident on the device (viwb_tracker_*): track() = FeatureTracker::trackImage() per stream.
    cam0 / cam1 = (fx, fy, cx, cy, k1, k2, p1, p2) (viwb_tracker_create) or, when either is a Camera, cameras of any model
    (viwb_tracker_create_camera; a tuple beside a Camera is taken as a pinhole Camera); cam1 None = mono sessions."""

    def __init__(self, ctx, streams, width, height, cam0, cam1=None, max_cnt=150, min_dist=30, flow_back=True):
        self.ctx, self.F, self.w, self.h, self.maxn, self.stereo = ctx, streams, width, height, max_cnt, cam1 is not None
        self.hnd = C.c_void_p()
        if isinstance(cam0, Camera) or isinstance(cam1, Camera):
            cams = [c if isinstance(c, Camera) else Camera.pinhole(*[float(v) for v in c]) for c in (cam0, cam1 if cam1 is not None else cam0)]
            cfg = TrackerConfig(max_cnt, int(min_dist), 1 if flow_back else 0, 1 if self.stereo else 0)
            ctx._ck(ctx.lib.viwb_tracker_create_camera(ctx.h, C.c_int(streams), C.c_int(width), C.c_int(height), C.byref(cfg), (Camera * 2)(*cams), C.byref(self.hnd)),
                    "viwb_tracker_create_camera")
        else:
            cfg = TrackerConfig(max_cnt, int(min_dist), 1 if flow_back else 0, 1 if self.stereo else 0,
                                (C.c_double * 16)(*([float(v) for v in cam0] + [float(v) for v in (cam1 if cam1 is not None else cam0)])))
            ctx._ck(ctx.lib.viwb_tracker_create(ctx.h, C.c_int(streams), C.c_int(width), C.c_int(height), C.byref(cfg), C.byref(self.hnd)), "viwb_tracker_create")
        self.n_left, self.n_right = np.zeros(streams, np.int32), np.zeros(streams, np.int32)
        self.ids, self.track_cnt, self.ids_right = (np.zeros((streams, max_cnt), np.int32) for _ in range(3))
        self.feat, self.feat_right = np.zeros((streams, max_cnt, 6), np.float32), np.zeros((streams, max_cnt, 6), np.float32)
        self._keep = None

    def _ptrs(self, imgs):
        assert imgs.dtype == np.uint8 and imgs.shape == (self.F, self.h, self.w) and imgs.strides[2] == 1
        return (C.c_void_p * self.F)(*[imgs.ctypes.data + f * imgs.strides[0] for f in range(self.F)]), int(imgs.strides[1])

    def track(self, cur_time, left, right=None, predict_pts=None, has_prediction=None):
        """asynchronous; call download() for the featureFrame rows"""
        pl, stride = self._ptrs(left)
        pr = None
        if self.stereo and right is not None:       # a missing right image is the C ABI's error to report
            pr, s2 = self._ptrs(right)
            assert s2 == stride
        pp = None if predict_pts is None else np.ascontiguousarray(predict_pts, np.float32)
        hp = None if has_prediction is None else np.ascontiguousarray(has_prediction, np.uint8)
        assert pp is None or (pp.shape == (self.F, self.maxn, 2) and hp is not None and hp.shape == (self.F,))
        self._keep = (left, right, pl, pr, pp, hp)
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        self.ctx._ck(self.ctx.lib.viwb_tracker_track(self.hnd, C.c_double(cur_time), pl, pr, C.c_int(stride), vp(pp), vp(hp)), "viwb_tracker_track")

    def feedback(self, remove_ids=None, predictions=None):
        """FeatureTracker::removeOutliers then setPrediction on every stream (estimator.cpp:841-843), asynchronous.
        remove_ids: per stream, an iterable of feature ids (or None for no removal at all).
        predictions: per stream, None (no prediction for that stream) or (ids, pts_cam [k, 3]) -- the valid rows of Context.predict_pts;
        the next track() consumes it and must be called without predict_pts."""
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        n_rm = rm = n_pr = pid = pts = hp = None
        if remove_ids is not None:
            assert len(remove_ids) == self.F
            lists = [np.asarray(list(r) if r is not None else [], np.int32).reshape(-1) for r in remove_ids]
            n_rm, rm = np.array([len(r) for r in lists], np.int32), np.ascontiguousarray(np.concatenate(lists), np.int32)
        if predictions is not None:
            assert len(predictions) == self.F
            hp = np.array([0 if p is None else 1 for p in predictions], np.uint8)
            idl = [np.zeros(0, np.int32) if p is None else np.asarray(p[0], np.int32).reshape(-1) for p in predictions]
            ptl = [np.zeros((0, 3)) if p is None else np.asarray(p[1], np.float64).reshape(-1, 3) for p in predictions]
            assert all(len(a) == len(b) for a, b in zip(idl, ptl))
            n_pr, pid, pts = np.array([len(a) for a in idl], np.int32), np.ascontiguousarray(np.concatenate(idl), np.int32), np.ascontiguousarray(np.concatenate(ptl), np.float64)
        self.ctx._ck(self.ctx.lib.viwb_tracker_feedback(self.hnd, vp(n_rm), vp(rm), vp(n_pr), vp(pid), vp(pts), vp(hp)), "viwb_tracker_feedback")

    def download(self):
        """-> per stream dicts are left to the caller; returns (n_left, ids, track_cnt, feat, n_right, ids_right, feat_right) views"""
        vp = lambda x: x.ctypes.data_as(C.c_void_p)
        self.ctx._ck(self.ctx.lib.viwb_tracker_download(self.hnd, vp(self.n_left), vp(self.ids), vp(self.track_cnt), vp(self.feat), vp(self.n_right) if self.stereo else None,
                                                        vp(self.ids_right) if self.stereo else None, vp(self.feat_right) if self.stereo else None), "viwb_tracker_download")
        return self.n_left, self.ids, self.track_cnt, self.feat, self.n_right, self.ids_right, self.feat_right

    def feature_frame(self, f):
        """featureFrame of stream f as the reference builds it: {feature_id: [(camera_id, [x, y, z, u, v, vx, vy]), ...]}"""
        out = {}
        for j in range(self.n_left[f]):
            x, y, u, v, vx, vy = (float(t) for t in self.feat[f, j])
            out.setdefault(int(self.ids[f, j]), []).append((0, [x, y, 1.0, u, v, vx, vy]))
        if self.stereo:
            for j in range(self.n_right[f]):
                x, y, u, v, vx, vy = (float(t) for t in self.feat_right[f, j])
                out.setdefault(int(self.ids_right[f, j]), []).append((1, [x, y, 1.0, u, v, vx, vy]))
        return out

    def algorithmic_bytes(self):
        return float(self.ctx.lib.viwb_tracker_algorithmic_bytes(self.hnd))

    def close(self):
        if self.hnd:
            self.ctx.lib.viwb_tracker_destroy(self.hnd)
            self.hnd = C.c_void_p()


class FeaturesConfig(C.Structure):
    _fields_ = [("max_rows", C.c_int), ("max_features", C.c_int), ("stereo", C.c_int), ("min_parallax", C.c_double), ("focal_length", C.c_double),
                ("init_depth", C.c_double)]


class Features:
    """`streams` FeatureManager lists resident on the device (viwb_features_*).  Per-stream arguments are sequences / arrays of length streams;
    states are [streams, 207] windows.  Errors raise ViwbError."""

    def __init__(self, ctx, streams, max_rows, stereo, min_parallax, focal_length=460.0, init_depth=5.0, max_features=0):
        self.ctx, self.F, self.R, self.stereo = ctx, streams, max_rows, bool(stereo)
        self.M = max_features or (abi.NUM_FRAMES * max_rows)
        self.hnd = C.c_void_p()
        cfg = FeaturesConfig(max_rows, max_features, 1 if stereo else 0, min_parallax, focal_length, init_depth)
        ctx._ck(ctx.lib.viwb_features_create(ctx.h, C.c_int(streams), C.byref(cfg), C.byref(self.hnd)), "viwb_features_create")

    def _call(self, name, *args):
        self.ctx._ck(getattr(self.ctx.lib, name)(self.hnd, *args), name)

    @staticmethod
    def _vp(x):
        return None if x is None else x.ctypes.data_as(C.c_void_p)

    def _per_stream(self, v, dtype):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype), (self.F,)), dtype)
        return a

    def add(self, frame_count, td, rows):
        """rows: per stream (ids, feat [n, 6]) or (ids, feat, ids_right, feat_right) -- the featureFrame of the tick"""
        R, F = self.R, self.F
        nl, nr = np.zeros(F, np.int32), np.zeros(F, np.int32)
        ids, idr = np.zeros((F, R), np.int32), np.zeros((F, R), np.int32)
        feat, fr = np.zeros((F, R, 6), np.float32), np.zeros((F, R, 6), np.float32)
        for s, row in enumerate(rows):
            a, b = np.asarray(row[0], np.int32).reshape(-1), np.asarray(row[1], np.float32).reshape(-1, 6)
            nl[s] = len(a)
            ids[s, : min(len(a), R)], feat[s, : min(len(a), R)] = a[:R], b[:R]
            if len(row) > 2 and row[2] is not None:
                c, d = np.asarray(row[2], np.int32).reshape(-1), np.asarray(row[3], np.float32).reshape(-1, 6)
                nr[s] = len(c)
                idr[s, : min(len(c), R)], fr[s, : min(len(c), R)] = c[:R], d[:R]
        fc, t = self._per_stream(frame_count, np.int32), self._per_stream(td, np.float64)
        vp = self._vp
        self._call("viwb_features_add", vp(fc), vp(t), vp(nl), vp(ids), vp(feat), vp(nr) if self.stereo else None, vp(idr), vp(fr))

    def add_tracked(self, tracker, frame_count, td):
        fc, t = self._per_stream(frame_count, np.int32), self._per_stream(td, np.float64)
        self._call("viwb_features_add_tracked", tracker.hnd, self._vp(fc), self._vp(t))

    def decisions(self):
        """-> dict of [streams] arrays: margin_flag, last_track_num, long_track_num, new_feature_num, last_average_parallax"""
        out = {k: np.zeros(self.F, np.int32) for k in ("margin_flag", "last_track_num", "long_track_num", "new_feature_num")}
        out["last_average_parallax"] = np.zeros(self.F)
        vp = self._vp
        self._call("viwb_features_decisions", vp(out["margin_flag"]), vp(out["last_track_num"]), vp(out["long_track_num"]), vp(out["new_feature_num"]),
                   vp(out["last_average_parallax"]))
        return out

    def triangulate(self, states):
        st = np.ascontiguousarray(states, np.float64).reshape(self.F, abi.STATE_FIXED)
        self._call("viwb_features_triangulate", self._vp(st))

    def window(self, vis_cap):
        """-> (tables, inv_depth, landmark_ids): tables[s] = the visual keyword arguments of abi.WindowProblem (num_landmarks, vis_type,
        vis_landmark, vis_frame_i, vis_frame_j, vis_obs); inv_depth[s] / landmark_ids[s] per landmark"""
        F, L = self.F, MAX_LANDMARKS
        nlm, nv = np.zeros(F, np.int32), np.zeros(F, np.int32)
        vt, vl, vi, vj = (np.zeros((F, max(vis_cap, 1)), np.int32) for _ in range(4))
        vo = np.zeros((F, max(vis_cap, 1), 12))
        inv, lid = np.zeros((F, L)), np.zeros((F, L), np.int32)
        vp = self._vp
        self._call("viwb_features_window", C.c_int(vis_cap), vp(nlm), vp(nv), vp(vt), vp(vl), vp(vi), vp(vj), vp(vo), vp(inv), vp(lid))
        tables = [dict(num_landmarks=int(nlm[s]), vis_type=vt[s, : nv[s]].copy(), vis_landmark=vl[s, : nv[s]].copy(), vis_frame_i=vi[s, : nv[s]].copy(),
                       vis_frame_j=vj[s, : nv[s]].copy(), vis_obs=vo[s, : nv[s]].copy()) for s in range(F)]
        return tables, [inv[s, : nlm[s]].copy() for s in range(F)], [lid[s, : nlm[s]].copy() for s in range(F)]

    def set_depth(self, inv_depth):
        """inv_depth: per stream, the landmarks' inverse depths in the last export's numbering"""
        x = np.zeros((self.F, MAX_LANDMARKS))
        for s, v in enumerate(inv_depth):
            v = np.asarray(v, np.float64).reshape(-1)
            x[s, : len(v)] = v
        self._call("viwb_features_set_depth", self._vp(x))

    def remove_outliers(self, outliers):
        """outliers: per stream, per-landmark flags of the last export -> per stream the removed ids, ascending"""
        x = np.zeros((self.F, MAX_LANDMARKS), np.uint8)
        for s, v in enumerate(outliers):
            v = np.asarray(v, np.uint8).reshape(-1)
            x[s, : len(v)] = v
        n, ids = np.zeros(self.F, np.int32), np.zeros((self.F, self.M), np.int32)
        self._call("viwb_features_remove_outliers", self._vp(x), self._vp(n), self._vp(ids))
        return [ids[s, : n[s]].copy() for s in range(self.F)]

    def predict(self, states, frame_count):
        """-> per stream None (frame_count < 2: no setPrediction) or (ids, pts_cam [k, 3]), the form Tracker.feedback takes"""
        st = np.ascontiguousarray(states, np.float64).reshape(self.F, abi.STATE_FIXED)
        fc = self._per_stream(frame_count, np.int32)
        n, ids, pts, hp = np.zeros(self.F, np.int32), np.zeros(self.F * self.M, np.int32), np.zeros((self.F * self.M, 3)), np.zeros(self.F, np.uint8)
        vp = self._vp
        self._call("viwb_features_predict", vp(st), vp(fc), vp(n), vp(ids), vp(pts), vp(hp))
        return self._predictions(n, ids, pts, hp)

    def _predictions(self, n, ids, pts, hp):
        out, o = [], 0
        for s in range(self.F):
            out.append((ids[o: o + n[s]].copy(), pts[o: o + n[s]].copy()) if hp[s] else None)
            o += n[s]
        return out

    def batch(self, problems, states, flags=None, options=None):
        """viwb_features_batch_create: one window per stream, its visual table and landmark inverse depths taken from the lists on the device.
        problems[s]: abi.WindowProblem with everything but the visual table (num_landmarks 0); states [streams, 207] -> a Batch whose download /
        outliers size each window by the landmark count the lists gave it (Batch.num_landmarks)."""
        assert len(problems) == self.F
        return Batch(self.ctx, problems, states, flags, options, features=self)

    def set_depth_from(self, batch):
        """setDepth from the batch's current landmark states (viwb_features_set_depth_batch)"""
        self._call("viwb_features_set_depth_batch", batch.h)

    def remove_outliers_from(self, batch, focal=460.0, thresh=3.0):
        """outliersRejection on the batch + removeOutlier (viwb_features_remove_outliers_batch) -> per stream the removed ids, ascending"""
        n, ids = np.zeros(self.F, np.int32), np.zeros((self.F, self.M), np.int32)
        self._call("viwb_features_remove_outliers_batch", batch.h, C.c_double(focal), C.c_double(thresh), self._vp(n), self._vp(ids))
        return [ids[s, : n[s]].copy() for s in range(self.F)]

    def predict_from(self, batch, frame_count):
        """predict() with each stream's fixed state read from the batch (viwb_features_predict_batch)"""
        fc = self._per_stream(frame_count, np.int32)
        n, ids, pts, hp = np.zeros(self.F, np.int32), np.zeros(self.F * self.M, np.int32), np.zeros((self.F * self.M, 3)), np.zeros(self.F, np.uint8)
        vp = self._vp
        self._call("viwb_features_predict_batch", batch.h, vp(fc), vp(n), vp(ids), vp(pts), vp(hp))
        return self._predictions(n, ids, pts, hp)

    def slide(self, frame_count, shift_depth, marg_R=None, marg_P=None, new_R=None, new_P=None):
        fc, sh = self._per_stream(frame_count, np.int32), self._per_stream(shift_depth, np.uint8)
        m = [None if a is None else np.ascontiguousarray(a, np.float64) for a in (marg_R, marg_P, new_R, new_P)]
        vp = self._vp
        self._call("viwb_features_slide", vp(fc), vp(sh), vp(m[0]), vp(m[1]), vp(m[2]), vp(m[3]))

    def remove_failures(self):
        self._call("viwb_features_remove_failures")

    def download(self):
        """-> per stream dict: ids, start_frame, num_obs, depth, solve_flag [n]; obs [n][11][12] float32; cur_td [n][11]; is_stereo [n][11]"""
        F, M = self.F, self.M
        n = np.zeros(F, np.int32)
        ids, sf, no, fl = (np.zeros((F, M), np.int32) for _ in range(4))
        dep = np.zeros((F, M))
        obs, td, ster = np.zeros((F, M, 11, 12), np.float32), np.zeros((F, M, 11)), np.zeros((F, M, 11), np.uint8)
        vp = self._vp
        self._call("viwb_features_download", vp(n), vp(ids), vp(sf), vp(no), vp(dep), vp(fl), vp(obs), vp(td), vp(ster))
        return [dict(ids=ids[s, : n[s]].copy(), start_frame=sf[s, : n[s]].copy(), num_obs=no[s, : n[s]].copy(), depth=dep[s, : n[s]].copy(),
                     solve_flag=fl[s, : n[s]].copy(), obs=obs[s, : n[s]].copy(), cur_td=td[s, : n[s]].copy(), is_stereo=ster[s, : n[s]].copy()) for s in range(F)]

    def close(self):
        if self.hnd:
            self.ctx.lib.viwb_features_destroy(self.hnd)
            self.hnd = C.c_void_p()


class Detector:
    """setMask + goodFeaturesToTrack for `streams` sessions per submission (viwb_detector_*).
    images: uint8 [streams, height, width] host array, or None with resident=<LkBatch> to use the tracker's current left images."""

    def __init__(self, ctx, streams, width, height, max_pts, min_dist):
        self.ctx, self.F, self.w, self.h, self.maxn = ctx, streams, width, height, max_pts
        self.hnd = C.c_void_p()
        ctx._ck(ctx.lib.viwb_detector_create(ctx.h, C.c_int(streams), C.c_int(width), C.c_int(height), C.c_int(max_pts), C.c_int(int(min_dist)), C.byref(self.hnd)),
                "viwb_detector_create")
        self.keep = np.zeros((streams, max_pts), np.int32)
        self.n_keep = np.zeros(streams, np.int32)
        self.new_pts = np.zeros((streams, max_pts, 2), np.float32)
        self.n_new = np.zeros(streams, np.int32)

    def detect(self, images, pts, track_cnt, n_pts, max_cnt, quality=0.01, resident=None, base_masks=None, want_mask=False):
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)
        ip, stride = None, self.w
        if images is not None:
            assert images.dtype == np.uint8 and images.shape == (self.F, self.h, self.w) and images.strides[2] == 1
            ip = (C.c_void_p * self.F)(*[images.ctypes.data + f * images.strides[0] for f in range(self.F)])
            stride = int(images.strides[1])
        bp = None
        if base_masks is not None:
            base_masks = np.ascontiguousarray(base_masks, np.uint8)
            assert base_masks.shape == (self.F, self.h, self.w)
            bp = (C.c_void_p * self.F)(*[base_masks.ctypes.data + f * base_masks.strides[0] for f in range(self.F)])
        p = np.ascontiguousarray(pts, np.float32); c = np.ascontiguousarray(track_cnt, np.int32); n = np.ascontiguousarray(n_pts, np.int32)
        assert p.shape == (self.F, self.maxn, 2) and c.shape == (self.F, self.maxn) and n.shape == (self.F,)
        mask = np.zeros((self.F, self.h, self.w), np.uint8) if want_mask else None
        self.ctx._ck(self.ctx.lib.viwb_detector_detect(self.hnd, ip, C.c_int(stride), resident.hnd if resident is not None else None, bp, vp(p), vp(c), vp(n),
                                                       C.c_int(max_cnt), C.c_double(quality), vp(self.keep), vp(self.n_keep), vp(self.new_pts), vp(self.n_new), vp(mask)),
                     "viwb_detector_detect")
        return self.keep, self.n_keep, self.new_pts, self.n_new, mask

    def algorithmic_bytes(self):
        return float(self.ctx.lib.viwb_detector_algorithmic_bytes(self.hnd))

    def close(self):
        if self.hnd:
            self.ctx.lib.viwb_detector_destroy(self.hnd)
            self.hnd = C.c_void_p()


class LkBatch:
    """One camera tick of `streams` independent sessions per submission (viwb_lk_batch_*).
    Images: uint8 arrays [streams, height, width] (C-contiguous); points: float32 [streams, max_points, 2]."""

    def __init__(self, ctx, streams, width, height, max_points, stereo=True, flow_back=True):
        self.ctx, self.F, self.w, self.h, self.maxn, self.stereo = ctx, streams, width, height, max_points, stereo
        self.hnd = C.c_void_p()
        ctx._ck(ctx.lib.viwb_lk_batch_create(ctx.h, C.c_int(streams), C.c_int(width), C.c_int(height), C.c_int(max_points), C.c_int(1 if stereo else 0),
                                             C.c_int(1 if flow_back else 0), C.byref(self.hnd)), "viwb_lk_batch_create")
        self.cur_pts = np.zeros((streams, max_points, 2), np.float32)
        self.right_pts = np.zeros((streams, max_points, 2), np.float32)
        self.status = np.zeros((streams, max_points), np.uint8)
        self.status_right = np.zeros((streams, max_points), np.uint8)
        self._keep = None

    def _ptrs(self, imgs):
        if imgs is None:
            return None, None
        assert imgs.dtype == np.uint8 and imgs.shape == (self.F, self.h, self.w) and imgs.strides[2] == 1
        arr = (C.c_void_p * self.F)(*[imgs.ctypes.data + f * imgs.strides[0] for f in range(self.F)])
        return arr, int(imgs.strides[1])

    def _marshal_upload(self, prev=None, cur=None, right=None, prev_pts=None, n_prev=None, stereo_pts=None, n_stereo=None):
        """(C arguments, objects that must outlive the asynchronous copies) of viwb_lk_batch_upload"""
        strides = set()
        pp, s0 = self._ptrs(prev); pc, s1 = self._ptrs(cur); pr, s2 = self._ptrs(right)
        for s in (s0, s1, s2):
            if s is not None:
                strides.add(s)
        assert len(strides) <= 1
        stride = strides.pop() if strides else self.w

        def f32(a):
            if a is None:
                return None
            a = np.ascontiguousarray(a, np.float32)
            assert a.shape == (self.F, self.maxn, 2)
            return a

        def i32(a):
            return None if a is None else np.ascontiguousarray(a, np.int32)
        a0, a1, c0, c1 = f32(prev_pts), f32(stereo_pts), i32(n_prev), i32(n_stereo)
        vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        return (self.hnd, pp, pc, pr, C.c_int(stride), vp(a0), vp(c0), vp(a1), vp(c1)), (prev, cur, right, a0, a1, c0, c1, pp, pc, pr)

    def upload(self, **kw):
        args, self._keep = self._marshal_upload(**kw)      # host buffers must outlive the asynchronous copies
        self.ctx._ck(self.ctx.lib.viwb_lk_batch_upload(*args), "viwb_lk_batch_upload")

    def prepare_upload(self, **kw):
        """upload() with the argument marshalling done once: returns a callable that only makes the C call (a camera driver hands over the same ring of
        page-locked buffers tick after tick; building F-entry pointer arrays in Python costs more than the call)."""
        args, keep = self._marshal_upload(**kw)

        def call():
            self._keep = keep
            self.ctx._ck(self.ctx.lib.viwb_lk_batch_upload(*args), "viwb_lk_batch_upload")
        return call

    def run(self):
        self.ctx._ck(self.ctx.lib.viwb_lk_batch_run(self.hnd), "viwb_lk_batch_run")

    def download(self):
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        self.ctx._ck(self.ctx.lib.viwb_lk_batch_download(self.hnd, vp(self.cur_pts), vp(self.status), vp(self.right_pts) if self.stereo else None,
                                                         vp(self.status_right) if self.stereo else None), "viwb_lk_batch_download")
        return self.cur_pts, self.status, self.right_pts, self.status_right

    def algorithmic_bytes(self):
        return float(self.ctx.lib.viwb_lk_batch_algorithmic_bytes(self.hnd))

    def close(self):
        if self.hnd:
            self.ctx.lib.viwb_lk_batch_destroy(self.hnd)
            self.hnd = C.c_void_p()


class Batch:
    """Device-resident batch of windows: upload once, run many times.  features: a Features whose lists supply the visual tables
    (viwb_features_batch_create; Features.batch), else viwb_batch_create with the problems' own."""

    def __init__(self, ctx, problems, states, flags=None, options=None, features=None):
        self.ctx = ctx
        self.B = len(problems)
        self.problems = problems
        self._arr = (abi.Problem * self.B)()
        for i, p in enumerate(problems):
            p.fill(self._arr[i])
        fl = (C.c_int32 * self.B)(*[int(f) for f in flags]) if flags is not None else None
        opt = options if options is not None else abi.default_options()
        self.h = C.c_void_p()
        if features is None:
            self._states = [np.ascontiguousarray(s, np.float64) for s in states]
            sp = (abi.c_double_p * self.B)(*[_dp(s) for s in self._states])
            self.num_landmarks = [p.num_landmarks for p in problems]
            ctx._ck(ctx.lib.viwb_batch_create(ctx.h, C.c_int(self.B), self._arr, sp, C.byref(opt), fl, C.byref(self.h)), "viwb_batch_create")
            return
        for i, p in enumerate(problems):          # the lists supply the visual tables: an empty one is passed as NULL
            if len(p.vis_type) == 0:
                a = self._arr[i]
                a.vis_type = a.vis_landmark = a.vis_frame_i = a.vis_frame_j = None
                a.vis_obs = None
        self._states = np.ascontiguousarray(np.asarray(states, np.float64).reshape(self.B, abi.STATE_FIXED))
        nlm = np.zeros(self.B, np.int32)
        features._call("viwb_features_batch_create", self._arr, _dp(self._states), C.byref(opt), fl, nlm.ctypes.data_as(C.c_void_p), C.byref(self.h))
        self.num_landmarks = [int(x) for x in nlm]

    def run(self):
        self.ctx._ck(self.ctx.lib.viwb_batch_run(self.ctx.h, self.h), "viwb_batch_run")

    def reset(self):
        """The windows as uploaded (viwb_batch_reset_states)."""
        self.ctx._ck(self.ctx.lib.viwb_batch_reset_states(self.ctx.h, self.h), "viwb_batch_reset_states")

    def algorithmic_bytes(self):
        return float(self.ctx.lib.viwb_batch_algorithmic_bytes(self.h))

    def solve_launch(self, occupancy=True):
        """(threads per block, dynamic shared-memory bytes, blocks per SM or None) of this batch's solve kernel (viwb_batch_solve_launch)."""
        nt, sm, bps = C.c_int(), C.c_int(), C.c_int()
        self.ctx._ck(self.ctx.lib.viwb_batch_solve_launch(self.ctx.h, self.h, C.byref(nt), C.byref(sm), C.byref(bps) if occupancy else None),
                     "viwb_batch_solve_launch")
        return nt.value, sm.value, (bps.value if occupancy else None)

    def download(self, want_priors=True):
        sts = [np.zeros(abi.STATE_FIXED + n) for n in self.num_landmarks]
        sp = (abi.c_double_p * self.B)(*[_dp(s) for s in sts])
        summ = (abi.Summary * self.B)()
        pri = [abi.PriorData() for _ in range(self.B)] if want_priors else None
        parr = None
        if want_priors:
            parr = (abi.Prior * self.B)()
            for i, p in enumerate(pri):
                parr[i] = p.c
        self.ctx._ck(self.ctx.lib.viwb_batch_download(self.ctx.h, self.h, sp, summ, parr), "viwb_batch_download")
        if want_priors:
            for i, p in enumerate(pri):
                p.c.valid, p.c.n, p.c.num_blocks = parr[i].valid, parr[i].n, parr[i].num_blocks
                for k in range(abi.NUM_FIXED_BLOCKS):
                    p.c.block_id[k], p.c.block_idx[k] = parr[i].block_id[k], parr[i].block_idx[k]
        return sts, list(summ), pri

    def outliers(self, focal=460.0, thresh=3.0):
        """Estimator::outliersRejection on the windows as the batch currently holds them (call after run())."""
        outs = [np.zeros(max(n, 1), np.uint8) for n in self.num_landmarks]
        arr = (C.c_void_p * self.B)(*[o.ctypes.data for o in outs])
        self.ctx._ck(self.ctx.lib.viwb_batch_outliers(self.ctx.h, self.h, C.c_double(focal), C.c_double(thresh), arr), "viwb_batch_outliers")
        return [o[:n] for o, n in zip(outs, self.num_landmarks)]

    def destroy(self):
        if self.h:
            self.ctx.lib.viwb_batch_destroy(self.ctx.h, self.h)
            self.h = C.c_void_p()
