// C++ node glue over the C-ABI: what a maintainer drops into aruco_detect / fiducial_slam instead of
// the OpenCV calls.  Header-only, no ROS headers: the message structs below mirror fiducial_msgs
// field-for-field so that, inside a ROS build, filling the real messages is a member-wise copy
// (see INTEGRATION.md).  Method names follow the reference node
// (aruco_detect/src/aruco_detect.cpp, fiducial_slam/src/fiducial_slam.cpp).
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <stdexcept>
#include <string>
#include <fstream>
#include <sstream>
#include <cstdio>
#include <cmath>
#include <vector>

#include "../../include/fiducials_b200.h"

namespace fid_glue {

struct Header {  // std_msgs/Header
    uint32_t seq = 0;
    uint32_t stamp_sec = 0, stamp_nsec = 0;
    std::string frame_id;
};
struct Fiducial {  // fiducial_msgs/msg/Fiducial.msg:3-14
    int32_t fiducial_id = 0;
    int32_t direction = 0;
    double x0 = 0, y0 = 0, x1 = 0, y1 = 0, x2 = 0, y2 = 0, x3 = 0, y3 = 0;
};
struct FiducialArray {  // FiducialArray.msg
    Header header;
    std::vector<Fiducial> fiducials;
};
struct Transform {  // geometry_msgs/Transform
    double tx = 0, ty = 0, tz = 0;
    double qx = 0, qy = 0, qz = 0, qw = 1;
};
struct FiducialTransform {  // FiducialTransform.msg:2-6
    int32_t fiducial_id = 0;
    Transform transform;
    double image_error = 0, object_error = 0, fiducial_area = 0;
};
struct FiducialTransformArray {  // FiducialTransformArray.msg:3-5
    Header header;
    int32_t image_seq = 0;
    std::vector<FiducialTransform> transforms;
};
struct ObjectHypothesisWithPose {  // vision_msgs, as aruco_detect.cpp:463-476 fills it
    int32_t id = 0;
    double score = 0;
    Transform pose;  // position + orientation
};
struct Detection2D {
    std::vector<ObjectHypothesisWithPose> results;
};
struct Detection2DArray {
    Header header;
    std::vector<Detection2D> detections;
};
struct FiducialMapEntry {  // FiducialMapEntry.msg:2-10
    int32_t fiducial_id = 0;
    double x = 0, y = 0, z = 0, rx = 0, ry = 0, rz = 0;
};
struct FiducialMapEntryArray {
    std::vector<FiducialMapEntry> fiducials;
};

inline void check(int status, const char* what) {
    if (status != FID_OK) throw std::runtime_error(std::string(what) + ": " + fid_strerror(status));
}

// aruco_detect's FiducialsNode, minus ROS transport.
class FiducialsNode {
   public:
    FiducialsNode(int dictionary, double fiducial_len_, int max_width, int max_height, int device = 0) : fiducial_len(fiducial_len_) {
        fid_params p;
        check(fid_default_params(&p), "fid_default_params");  // aruco_detect.cpp:690-727
        p.dictionary = dictionary;                            // :611
        check(fid_create(&p, device, max_width, max_height, 1, &det), "fid_create");
        specs.push_back(fid_dictionary_spec{dictionary, 0, 0.0});
    }

    // Further dictionaries after `dictionary` (new, no reference counterpart; a ROS binding would read them from parameters next to
    // `dictionary`): each with an id offset, so the published fiducial_id is id + id_offset, and a marker length (0 = fiducial_len).
    // The messages, ignoreIds and fiducialLens then use published ids.  Detection is detectMarkersMultiDict (fid_detect_multi_dict).
    void setDictionaries(const std::vector<fid_dictionary_spec>& extra) {
        std::vector<fid_dictionary_spec> all(1, specs[0]);
        all.insert(all.end(), extra.begin(), extra.end());
        check(fid_set_dictionaries(det, (int)all.size(), all.data()), "fid_set_dictionaries");
        specs = all;
    }
    // Detection on a downscaled frame (new, no reference counterpart; the reference's configCallback has no such field):
    // cv2's useAruco3Detection with minMarkerLengthRatioOriginalImg = ratio and minSideLengthCanonicalImg = min_side.  imageCallback
    // and poseEstimateCallback then work on the full-resolution corners the mode returns.  Not with several dictionaries.
    void setAruco3(double ratio, int min_side) {
        const fid_aruco3_params a{1, min_side, ratio};
        check(fid_set_aruco3(det, &a), "fid_set_aruco3");
    }
    // White-on-black markers too (new, no reference counterpart): cv2's detectInvertedMarker.  A group of nested outlines then keeps
    // its smallest, as in cv2, so black markers come back with other corners than without the flag.
    void setDetectInvertedMarker(bool enable) { check(fid_set_detect_inverted_marker(det, enable ? 1 : 0), "fid_set_detect_inverted_marker"); }
    ~FiducialsNode() {
        if (det) fid_destroy(det);
    }
    FiducialsNode(const FiducialsNode&) = delete;
    FiducialsNode& operator=(const FiducialsNode&) = delete;

    // configCallback, aruco_detect.cpp:257-298: the dynamic_reconfigure fields map one to one onto fid_params; the two booleans
    // select the corner refinement method as the reference does (:274-281, same rule at start-up :700-711)
    void configCallback(fid_params p, bool doCornerRefinement, bool cornerRefinementSubpix) {
        p.cornerRefinementMethod = doCornerRefinement ? (cornerRefinementSubpix ? 1 /* SUBPIX */ : 2 /* CONTOUR */) : 0 /* NONE */;
        check(fid_set_params(det, &p), "fid_set_params");  // replaces the first dictionary, keeps the others
        specs[0].dictionary = p.dictionary;
    }

    // camInfoCallback, aruco_detect.cpp:307-330
    void camInfoCallback(const double K[9], const double* D, int nD, const std::string& frame_id) {
        if (haveCamInfo) return;
        bool all_zero = true;
        for (int i = 0; i < 9; i++) all_zero = all_zero && K[i] == 0.0;
        if (all_zero) return;  // :313
        for (int i = 0; i < 9; i++) cam.K[i] = K[i];
        for (int i = 0; i < 5; i++) cam.D[i] = i < nD ? D[i] : 0.0;  // :317-323
        haveCamInfo = true;
        frameId = frame_id;
    }

    // imageCallback, aruco_detect.cpp:332-395: bgr = cv_bridge::toCvCopy(msg, BGR8) pixels (:348)
    bool imageCallback(const uint8_t* bgr, int width, int height, size_t stride, const Header& hdr, FiducialArray* fva) {
        if (!enable_detections) return false;  // :334
        fva->header = hdr;
        fva->header.frame_id = frameId;
        fva->fiducials.clear();
        ids.assign(FID_MAX_MARKERS, 0);
        corners.assign(FID_MAX_MARKERS * 8, 0.f);
        dictIdx.assign(FID_MAX_MARKERS, 0);
        int n = 0;
        const int rc = specs.size() > 1 ? fid_detect_multi_dict(det, bgr, width, height, stride, FID_MAX_MARKERS, &n, ids.data(), corners.data(), dictIdx.data())
                                        : fid_detect(det, bgr, width, height, stride, FID_MAX_MARKERS, &n, ids.data(), corners.data());
        if (rc != FID_OK) return false;  // frame dropped (:389-394)
        ids.resize(n);
        corners.resize((size_t)n * 8);
        dictIdx.resize(n);
        for (int i = 0; i < n; i++) {
            const int pub = ids[i] + specs[dictIdx[i]].id_offset;
            if (std::count(ignoreIds.begin(), ignoreIds.end(), pub) != 0) continue;  // :359-364
            Fiducial f;
            f.fiducial_id = pub;
            const float* c = &corners[(size_t)i * 8];
            f.x0 = c[0]; f.y0 = c[1]; f.x1 = c[2]; f.y1 = c[3]; f.x2 = c[4]; f.y2 = c[5]; f.x3 = c[6]; f.y3 = c[7];  // :366-376
            fva->fiducials.push_back(f);
        }
        last = hdr;
        return true;
    }

    // poseEstimateCallback, aruco_detect.cpp:397-538 (uses the member ids/corners like the reference)
    bool poseEstimateCallback(FiducialTransformArray* fta) {
        fta->header = last;
        fta->header.frame_id = frameId;
        fta->image_seq = (int32_t)last.seq;
        fta->transforms.clear();
        frameNum++;
        if (!doPoseEstimation) return true;
        if (!haveCamInfo) return false;  // :417-422
        std::vector<int32_t> oi;
        std::vector<double> ol;
        for (auto& kv : fiducialLens) {  // :239-244
            oi.push_back(kv.first);
            ol.push_back(kv.second);
        }
        // one fid_pose per dictionary, on its markers' published ids and its length (one call over all markers with one dictionary)
        std::vector<fid_transform> out(ids.size());
        for (size_t d = 0; d < specs.size(); d++) {
            std::vector<int32_t> gi, pos;
            std::vector<float> gc;
            for (size_t i = 0; i < ids.size(); i++) {
                if (dictIdx[i] != (int)d) continue;
                pos.push_back((int32_t)i);
                gi.push_back(ids[i] + specs[d].id_offset);
                gc.insert(gc.end(), corners.begin() + i * 8, corners.begin() + i * 8 + 8);
            }
            if (gi.empty()) continue;
            std::vector<fid_transform> g(gi.size());
            const double len = specs[d].fiducial_len > 0 ? specs[d].fiducial_len : fiducial_len;
            if (fid_pose(det, (int)gi.size(), gi.data(), gc.data(), &cam, len, (int)oi.size(), oi.data(), ol.data(), g.data()) != FID_OK) return true;
            for (size_t k = 0; k < pos.size(); k++) out[pos[k]] = g[k];
        }
        for (const fid_transform& t : out) {
            if (std::count(ignoreIds.begin(), ignoreIds.end(), t.fiducial_id) != 0) continue;  // :440
            FiducialTransform ft;
            ft.fiducial_id = t.fiducial_id;
            ft.transform = Transform{t.translation[0], t.translation[1], t.translation[2], t.rotation[0], t.rotation[1], t.rotation[2], t.rotation[3]};
            ft.image_error = t.image_error;
            ft.object_error = t.object_error;
            ft.fiducial_area = t.fiducial_area;
            fta->transforms.push_back(ft);
        }
        return true;
    }

    // vis_msgs variant (aruco_detect.cpp:403,462-478,534): vision_msgs/Detection2DArray with score = exp(-2 object_error)
    bool poseEstimateCallbackVis(Detection2DArray* vma) {
        FiducialTransformArray fta;
        if (!poseEstimateCallback(&fta)) return false;
        vma->header = fta.header;
        vma->detections.clear();
        for (const FiducialTransform& ft : fta.transforms) {
            Detection2D d;
            d.results.push_back(ObjectHypothesisWithPose{ft.fiducial_id, exp(-2.0 * ft.object_error), ft.transform});
            vma->detections.push_back(d);
        }
        return true;
    }

    double fiducial_len;
    bool doPoseEstimation = true, enable_detections = true, haveCamInfo = false;
    std::vector<int> ignoreIds;              // :540-571
    std::map<int, double> fiducialLens;      // :627-660
    std::string frameId;
    int frameNum = 0;

   private:
    fid_detector* det = nullptr;
    fid_camera cam{};
    std::vector<int32_t> ids;
    std::vector<float> corners;
    std::vector<int32_t> dictIdx;            // each marker's dictionary (all 0 with one dictionary)
    std::vector<fid_dictionary_spec> specs;  // entry 0 = the constructor's dictionary
    Header last;
};

// tf2 LinearMath pieces of the published pose (setRotation / getRotation / getRPY's yaw)
inline void tf2_q_to_m(const double q[4], double m[9]) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double s = 2.0 / (x * x + y * y + z * z + w * w);
    const double xs = x * s, ys = y * s, zs = z * s, wx = w * xs, wy = w * ys, wz = w * zs, xx = x * xs, xy = x * ys, xz = x * zs, yy = y * ys, yz = y * zs, zz = z * zs;
    const double r[9] = {1.0 - (yy + zz), xy - wz, xz + wy, xy + wz, 1.0 - (xx + zz), yz - wx, xz - wy, yz + wx, 1.0 - (xx + yy)};
    for (int i = 0; i < 9; i++) m[i] = r[i];
}
inline void tf2_m_to_q(const double m[9], double q[4]) {
    const double tr = m[0] + m[4] + m[8];
    if (tr > 0.0) {
        double s = sqrt(tr + 1.0);
        q[3] = s * 0.5;
        s = 0.5 / s;
        q[0] = (m[7] - m[5]) * s;
        q[1] = (m[2] - m[6]) * s;
        q[2] = (m[3] - m[1]) * s;
    } else {
        const int i = m[0] < m[4] ? (m[4] < m[8] ? 2 : 1) : (m[0] < m[8] ? 2 : 0);
        const int j = (i + 1) % 3, k = (i + 2) % 3;
        double s = sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
        q[i] = s * 0.5;
        s = 0.5 / s;
        q[3] = (m[k * 3 + j] - m[j * 3 + k]) * s;
        q[j] = (m[j * 3 + i] + m[i * 3 + j]) * s;
        q[k] = (m[k * 3 + i] + m[i * 3 + k]) * s;
    }
}
inline double tf2_get_yaw(const double m[9]) {  // third angle of tf2::Matrix3x3::getRPY
    if (fabs(m[6]) >= 1.0) return 0.0;
    const double c = cos(-asin(m[6]));
    return atan2(m[3] / c, m[0] / c);
}

// fiducial_slam's FiducialSlam + Map, minus ROS transport and tf (the two tf lookups of
// Map::updatePose, map.cpp:258-273, are passed in by the caller; nullptr = lookup failed).
class FiducialSlam {
   public:
    explicit FiducialSlam(int max_fiducials = 512, int device = 0) {
        fid_map_params p;
        check(fid_map_default_params(&p), "fid_map_default_params");
        p.max_fiducials = max_fiducials;
        check(fid_map_create(&p, device, &map), "fid_map_create");
        cap = max_fiducials;
    }
    ~FiducialSlam() {
        if (map) fid_map_destroy(map);
    }
    FiducialSlam(const FiducialSlam&) = delete;
    FiducialSlam& operator=(const FiducialSlam&) = delete;

    // transformCallback, fiducial_slam.cpp:79-105 + Map::update, map.cpp:152-176
    bool transformCallback(const FiducialTransformArray& msg, const fid_tf* T_baseCam, const fid_tf* T_camBase, fid_robot_pose* robot) {
        std::vector<fid_transform> obs(msg.transforms.size());
        for (size_t i = 0; i < obs.size(); i++) {
            const FiducialTransform& ft = msg.transforms[i];
            fid_transform& o = obs[i];
            o.fiducial_id = ft.fiducial_id;
            o.translation[0] = ft.transform.tx; o.translation[1] = ft.transform.ty; o.translation[2] = ft.transform.tz;
            o.rotation[0] = ft.transform.qx; o.rotation[1] = ft.transform.qy; o.rotation[2] = ft.transform.qz; o.rotation[3] = ft.transform.qw;
            o.image_error = ft.image_error; o.object_error = ft.object_error; o.fiducial_area = ft.fiducial_area;
        }
        return fid_map_update(map, 0, (int)obs.size(), obs.data(), T_baseCam, T_camBase, robot) == FID_OK;
    }

    // add_fiducial service (addFiducialCallback, map.cpp:821-828; handled by the next update, handleAddFiducial :489-535).
    // T_mapBase = the tf lookup map -> base, nullptr when it fails.
    bool addFiducial(int fiducial_id, const fid_tf* T_mapBase) { return fid_map_add_fiducial(map, 0, fiducial_id, T_mapBase) == FID_OK; }

    // ---- published pose: host-side message packing of updatePose's tail (map.cpp:337-379) ----
    bool overridePublishedCovariance = false;  // rosparam covariance_diagonal, map.cpp:110-125
    double covarianceDiagonal[6] = {0, 0, 0, 0, 0, 0};
    bool publish_6dof_pose = false;            // map.cpp:107
    // six values, all non-zero, or the parameter is ignored (map.cpp:112-124)
    void setCovarianceDiagonal(const std::vector<double>& d) {
        overridePublishedCovariance = d.size() == 6;
        for (size_t i = 0; i < 6; i++) covarianceDiagonal[i] = overridePublishedCovariance ? d[i] : 0.0;
        for (size_t i = 0; overridePublishedCovariance && i < 6; i++)
            if (d[i] == 0) {
                overridePublishedCovariance = false;
                for (double& v : covarianceDiagonal) v = 0.0;
            }
    }
    // covariance of the PoseWithCovarianceStamped on /fiducial_pose: toPose (transform_with_variance.h:69-84) + override (:341-345)
    void robotPoseCovariance(const fid_robot_pose& robot, double cov[36]) const {
        for (int i = 0; i < 36; i++) cov[i] = 0.0;
        for (int i = 0; i < 6; i++) cov[i * 6 + i] = overridePublishedCovariance ? covarianceDiagonal[i] : robot.variance;
    }
    // the transform broadcast as map -> odom (T_odomBase given) or map -> base: basePose * odom^-1 (:351-365), squashed to
    // x, y, yaw unless publish_6dof_pose (:369-379)
    Transform poseTf(const fid_robot_pose& robot, const fid_tf* T_odomBase) const {
        double R[9], t[3] = {robot.t[0], robot.t[1], robot.t[2]};
        tf2_q_to_m(robot.q, R);
        if (T_odomBase) {
            double Ro[9], Ri[9], ti[3], Rn[9];
            tf2_q_to_m(T_odomBase->q, Ro);
            for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++) Ri[i * 3 + j] = Ro[j * 3 + i];
            for (int i = 0; i < 3; i++) ti[i] = Ri[i * 3] * -T_odomBase->t[0] + Ri[i * 3 + 1] * -T_odomBase->t[1] + Ri[i * 3 + 2] * -T_odomBase->t[2];
            for (int i = 0; i < 3; i++) {
                for (int j = 0; j < 3; j++) Rn[i * 3 + j] = R[i * 3] * Ri[j] + R[i * 3 + 1] * Ri[3 + j] + R[i * 3 + 2] * Ri[6 + j];
                t[i] = (R[i * 3] * ti[0] + R[i * 3 + 1] * ti[1] + R[i * 3 + 2] * ti[2]) + robot.t[i];
            }
            for (int i = 0; i < 9; i++) R[i] = Rn[i];
        }
        if (!publish_6dof_pose) {
            t[2] = 0.0;
            const double yaw = tf2_get_yaw(R);
            const double ch = cos(yaw), sh = sin(yaw);  // setRPY(0, 0, yaw)
            const double Rz[9] = {ch, -sh, 0, sh, ch, 0, 0, 0, 1};
            for (int i = 0; i < 9; i++) R[i] = Rz[i];
        }
        double q[4];
        tf2_m_to_q(R, q);
        return Transform{t[0], t[1], t[2], q[0], q[1], q[2], q[3]};
    }

    // ---- localization against the map (new, no reference counterpart; fid_map_localize) ----
    // The /fiducial_vertices message (aruco_detect.cpp:358-379: ids and the float32 corners as float64) and the latched CameraInfo
    // (K, first five plumb_bob D) give the camera pose that all visible mapped markers determine together, with its covariance.
    // fiducial_len / overrides as the detector node uses them; T_camBase = the tf lookup camera -> base (nullptr: the camera's pose).
    fid_localization localize(const FiducialArray& vertices, const fid_camera& cam, double fiducial_len, const std::map<int, double>& overrides,
                              const fid_tf* T_camBase, double max_entry_variance = -1.0) {
        const int n = (int)vertices.fiducials.size();
        std::vector<int32_t> ids(std::max(n, 1), -1);
        std::vector<float> corners(8 * (size_t)std::max(n, 1), 0.f);
        for (int i = 0; i < n; i++) {
            const Fiducial& v = vertices.fiducials[i];
            ids[i] = v.fiducial_id;
            const double c[8] = {v.x0, v.y0, v.x1, v.y1, v.x2, v.y2, v.x3, v.y3};
            for (int k = 0; k < 8; k++) corners[8 * (size_t)i + k] = (float)c[k];
        }
        std::vector<int32_t> ov_ids;
        std::vector<double> ov_lens;
        for (const auto& kv : overrides) {
            ov_ids.push_back(kv.first);
            ov_lens.push_back(kv.second);
        }
        const int32_t count = n;
        fid_localization out;
        check(fid_map_localize(map, 0, 1, &count, ids.data(), corners.data(), std::max(n, 1), &cam, fiducial_len, (int)ov_ids.size(), ov_ids.data(), ov_lens.data(),
                               max_entry_variance, T_camBase, &out),
              "fid_map_localize");
        return out;
    }
    double multiErrorThreshold = -1.0;  // rosparam multi_error_theshold, map.cpp:127-129 (-1: never switches)
    // What goes on /fiducial_pose: the joint pose and its covariance when multiErrorThreshold >= 0, loc->status == FID_LOC_POSE and
    // loc->object_error < multiErrorThreshold; otherwise the fold's pose with robotPoseCovariance.  covariance_diagonal overrides
    // the diagonal of either (map.cpp:341-345).  Publication only: the fold and the map are unchanged.
    Transform publishedPose(const fid_robot_pose& robot, const fid_localization* loc, double cov[36]) const {
        if (loc && multiErrorThreshold >= 0 && loc->status == FID_LOC_POSE && loc->object_error < multiErrorThreshold) {
            for (int i = 0; i < 36; i++) cov[i] = loc->covariance[i];
            for (int i = 0; overridePublishedCovariance && i < 6; i++) cov[i * 6 + i] = covarianceDiagonal[i];
            return Transform{loc->t[0], loc->t[1], loc->t[2], loc->q[0], loc->q[1], loc->q[2], loc->q[3]};
        }
        robotPoseCovariance(robot, cov);
        return Transform{robot.t[0], robot.t[1], robot.t[2], robot.q[0], robot.q[1], robot.q[2], robot.q[3]};
    }

    // publishMap, map.cpp:629-654
    FiducialMapEntryArray publishMap() {
        std::vector<fid_map_entry> e(cap);
        int n = 0;
        check(fid_map_entries(map, 0, cap, &n, e.data()), "fid_map_entries");
        FiducialMapEntryArray out;
        for (int i = 0; i < n; i++) out.fiducials.push_back(FiducialMapEntry{e[i].fiducial_id, e[i].x, e[i].y, e[i].z, e[i].rx, e[i].ry, e[i].rz});
        return out;
    }

    // Map::saveMap, map.cpp:541-566
    bool saveMap(const std::string& filename) {
        std::vector<fid_map_entry> e(cap);
        int n = 0, np = 0;
        check(fid_map_entries(map, 0, cap, &n, e.data()), "fid_map_entries");
        std::vector<int32_t> pairs;
        fid_map_links(map, 0, 0, &np, nullptr);  // FID_ERR_CAPACITY by design: this call only asks for the count
        pairs.resize(2 * (size_t)np + 2);
        check(fid_map_links(map, 0, np, &np, pairs.data()), "fid_map_links");
        FILE* fp = fopen(filename.c_str(), "w");
        if (fp == NULL) return false;
        for (int i = 0; i < n; i++) {
            fprintf(fp, "%d %lf %lf %lf %lf %lf %lf %lf %d", e[i].fiducial_id, e[i].x, e[i].y, e[i].z, e[i].rx * 180.0 / M_PI, e[i].ry * 180.0 / M_PI, e[i].rz * 180.0 / M_PI,
                    e[i].variance, e[i].num_obs);
            for (int k = 0; k < np; k++)
                if (pairs[2 * k] == e[i].fiducial_id) fprintf(fp, " %d", pairs[2 * k + 1]);
            fprintf(fp, "\n");
        }
        fclose(fp);
        return true;
    }

    // Map::loadMap(filename), map.cpp:572-625: one fiducial per line, nine leading fields (id, x y z, roll pitch yaw
    // in degrees, variance, numObs), then the linked ids up to a tab or the end of the line; a line whose nine
    // fields do not parse is skipped (the reference logs "Invalid line").
    bool loadMap(const std::string& filename) {
        std::ifstream in(filename);
        if (!in) return false;
        std::vector<fid_map_file_entry> rows;
        std::vector<int32_t> pairs;
        std::string line;
        while (std::getline(in, line)) {
            // sscanf("%d %lf %lf %lf %lf %lf %lf %lf %d%[^\t\n]"): the nine numbers may be separated by any white space (tabs
            // included); only the link list that follows them ends at the first tab
            std::istringstream fields(line);
            fid_map_file_entry r{};
            if (!(fields >> r.fiducial_id >> r.x >> r.y >> r.z >> r.roll_deg >> r.pitch_deg >> r.yaw_deg >> r.variance >> r.num_obs)) continue;
            rows.push_back(r);
            std::string rest;
            std::getline(fields, rest);
            std::istringstream links(rest.substr(0, rest.find('\t')));
            for (int32_t linked; links >> linked;) {
                pairs.push_back(r.fiducial_id);
                pairs.push_back(linked);
            }
        }
        if (fid_map_load(map, 0, (int)rows.size(), rows.data()) != FID_OK) return false;
        return fid_map_add_links(map, 0, (int)pairs.size() / 2, pairs.data()) == FID_OK;
    }

   private:
    fid_map* map = nullptr;
    int cap = 0;
};

}  // namespace fid_glue
