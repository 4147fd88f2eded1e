// ref_features_glue.cpp -- TEST INFRASTRUCTURE ONLY.  C entry points that drive the reference's OWN FeatureManager
// (estimator/feature_manager.cpp, compiled unmodified into _ref/libviw_ref.so) through a scripted sequence of calls: addFeatureCheckParallax
// with image maps built from featureFrame rows, triangulate, setDepth, removeOutlier, removeBackShiftDepth / removeBack / removeFront,
// removeFailures, and a dump of the list.  Built by oracle/features.mk into _ref/libviw_ref_features.so; nothing of the reference is restated.
#include "estimator/feature_manager.h"
#include <map>
#include <set>
#include <vector>

namespace {
struct Session {
    Eigen::Matrix3d Rs[WINDOW_SIZE + 1];
    FeatureManager *fm;
    int stereo; double min_parallax, init_depth;
    void globals() const { STEREO = stereo; NUM_OF_CAM = stereo ? 2 : 1; MIN_PARALLAX = min_parallax; INIT_DEPTH = init_depth; }
};
Eigen::Quaterniond quat_at(const double *q) { return Eigen::Quaterniond(q[3], q[0], q[1], q[2]); }
Eigen::Matrix3d mat_at(const double *m) { Eigen::Matrix3d R; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R(r, c) = m[3 * r + c]; return R; }
Eigen::Matrix<double, 7, 1> row7(const float *f) {
    Eigen::Matrix<double, 7, 1> v;
    v << f[0], f[1], 1.0, f[2], f[3], f[4], f[5];                    // z = 1, as every featureFrame producer of the reference sets it
    return v;
}
}  // namespace

extern "C" void *ref_fm_create(int stereo, double min_parallax, double init_depth) {
    Session *s = new Session();
    s->stereo = stereo; s->min_parallax = min_parallax; s->init_depth = init_depth;
    s->globals();
    s->fm = new FeatureManager(s->Rs);
    return s;
}
extern "C" void ref_fm_destroy(void *h) { Session *s = (Session *)h; delete s->fm; delete s; }

// rows as in viwb_features_add (feat: x y p_u p_v v_x v_y); stats = keyframe, last_track_num, long_track_num, new_feature_num; *avg = last_average_parallax
extern "C" void ref_fm_add(void *h, int frame_count, double td, int n, const int32_t *ids, const float *feat, int nr, const int32_t *ids_r, const float *feat_r,
                           int32_t *stats, double *avg) {
    Session *s = (Session *)h; s->globals();
    std::map<int, std::vector<std::pair<int, Eigen::Matrix<double, 7, 1>>>> image;
    for (int i = 0; i < n; i++) image[ids[i]].emplace_back(0, row7(feat + 6 * i));
    for (int i = 0; i < nr; i++) image[ids_r[i]].emplace_back(1, row7(feat_r + 6 * i));
    stats[0] = s->fm->addFeatureCheckParallax(frame_count, image, td) ? 1 : 0;
    stats[1] = s->fm->last_track_num; stats[2] = s->fm->long_track_num; stats[3] = s->fm->new_feature_num; *avg = s->fm->last_average_parallax;
}
// state: the window of include/viwb.h (poses 7 x 11, extrinsics of cameras 0 / 1 at 176 / 183)
extern "C" void ref_fm_triangulate(void *h, int frame_count, const double *state) {
    Session *s = (Session *)h; s->globals();
    Eigen::Vector3d Ps[WINDOW_SIZE + 1], tic[2]; Eigen::Matrix3d Rs[WINDOW_SIZE + 1], ric[2];
    for (int i = 0; i <= WINDOW_SIZE; i++) { Ps[i] = Eigen::Vector3d(state[7 * i], state[7 * i + 1], state[7 * i + 2]); Rs[i] = quat_at(state + 7 * i + 3).toRotationMatrix(); }
    for (int c = 0; c < 2; c++) { tic[c] = Eigen::Vector3d(state[176 + 7 * c], state[177 + 7 * c], state[178 + 7 * c]); ric[c] = quat_at(state + 179 + 7 * c).toRotationMatrix(); }
    s->fm->triangulate(frame_count, Ps, Rs, tic, ric);
}
extern "C" void ref_fm_set_depth(void *h, int n, const double *x) {
    Session *s = (Session *)h; s->globals();
    Eigen::VectorXd v(n);
    for (int i = 0; i < n; i++) v(i) = x[i];
    s->fm->setDepth(v);
}
extern "C" void ref_fm_remove_outlier(void *h, int n, const int32_t *ids) {
    Session *s = (Session *)h; s->globals();
    std::set<int> idx(ids, ids + n);
    s->fm->removeOutlier(idx);
}
// R row-major camera-to-world, P [3]
extern "C" void ref_fm_remove_back_shift_depth(void *h, const double *marg_R, const double *marg_P, const double *new_R, const double *new_P) {
    Session *s = (Session *)h; s->globals();
    s->fm->removeBackShiftDepth(mat_at(marg_R), Eigen::Vector3d(marg_P[0], marg_P[1], marg_P[2]), mat_at(new_R), Eigen::Vector3d(new_P[0], new_P[1], new_P[2]));
}
extern "C" void ref_fm_remove_back(void *h) { Session *s = (Session *)h; s->globals(); s->fm->removeBack(); }
extern "C" void ref_fm_remove_front(void *h, int frame_count) { Session *s = (Session *)h; s->globals(); s->fm->removeFront(frame_count); }
extern "C" void ref_fm_remove_failures(void *h) { Session *s = (Session *)h; s->globals(); s->fm->removeFailures(); }
extern "C" int ref_fm_size(void *h) { return (int)((Session *)h)->fm->feature.size(); }
// the list in viwb_features_download's per-stream layout (obs narrowed back to the floats the rows came from)
extern "C" void ref_fm_dump(void *h, int32_t *ids, int32_t *start, int32_t *nobs, double *depth, int32_t *flag, float *obs, double *td, uint8_t *ster) {
    Session *s = (Session *)h;
    int k = 0;
    for (auto &f : s->fm->feature) {
        ids[k] = f.feature_id; start[k] = f.start_frame; nobs[k] = (int)f.feature_per_frame.size(); depth[k] = f.estimated_depth; flag[k] = f.solve_flag;
        for (int j = 0; j < 11; j++) {
            float *o = obs + ((size_t)k * 11 + j) * 12;
            for (int c = 0; c < 12; c++) o[c] = 0.f;
            td[k * 11 + j] = 0.0; ster[k * 11 + j] = 0;
            if (j >= (int)f.feature_per_frame.size()) continue;
            const FeaturePerFrame &p = f.feature_per_frame[j];
            const double v[12] = {p.point.x(), p.point.y(), p.uv.x(), p.uv.y(), p.velocity.x(), p.velocity.y(),
                                  p.pointRight.x(), p.pointRight.y(), p.uvRight.x(), p.uvRight.y(), p.velocityRight.x(), p.velocityRight.y()};
            for (int c = 0; c < (p.is_stereo ? 12 : 6); c++) o[c] = (float)v[c];
            td[k * 11 + j] = p.cur_td; ster[k * 11 + j] = p.is_stereo ? 1 : 0;
        }
        k++;
    }
}
