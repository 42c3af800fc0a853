// C interface around the REFERENCE's own Map class (fiducial_slam/src/map.cpp + transform_with_variance.cpp, compiled unmodified
// from the reference checkout against the stand-in headers of oracle/ref_shim -- see oracle/ref_shim/README.md and oracle/Makefile).
//
// TEST INFRASTRUCTURE ONLY: the compiled reference is the checker for oracle/slam_oracle.py (tests/test_map_ref.py) and for the CUDA
// map update (tests/test_gpu_slam.py), and the CPU arm of `bench.py --workload C5`.  Nothing here is linked into the product.
//
// The only reference logic restated in this file is FiducialSlam::transformCallback (fiducial_slam/src/fiducial_slam.cpp:79-105):
// a FiducialTransformArray becomes a vector<Observation> with variance = weighting_scale * object_error (or / fiducial_area).
#include <fiducial_slam/map.h>

#include <cstring>
#include <memory>

namespace {
struct MapRef {
    ros::NodeHandle nh;
    std::unique_ptr<Map> map;
    double weighting_scale = 1e9;
    bool use_area = false;
};
}  // namespace

extern "C" {

// cov_diag: 6 values or NULL; odom_frame "" disables the map -> odom composition (map.cpp:355-371)
void* mapref_create(double weighting_scale, int use_area, int read_only, int publish_6dof_pose, const double* cov_diag, const char* map_file, const char* odom_frame,
                    const char* base_frame) {
    MapRef* h = new MapRef();
    h->weighting_scale = weighting_scale;
    h->use_area = use_area != 0;
    h->nh.str["map_file"] = map_file;
    h->nh.str["odom_frame"] = odom_frame;
    h->nh.str["base_frame"] = base_frame;
    h->nh.num["read_only_map"] = read_only;
    h->nh.num["publish_6dof_pose"] = publish_6dof_pose;
    h->nh.num["publish_tf"] = 1;
    h->nh.num["systematic_error"] = 0.01;  // the static in map.cpp is shared by every Map of the process: always the default
    if (cov_diag) h->nh.vec["covariance_diagonal"] = std::vector<double>(cov_diag, cov_diag + 6);
    h->map.reset(new Map(h->nh));
    return h;
}

void mapref_destroy(void* p) { delete static_cast<MapRef*>(p); }

void mapref_clear_tf() { tf2_ros::TfTable::get().t.clear(); }

// lookupTransform(target, source): t7 = x y z qx qy qz qw
void mapref_set_tf(const char* target, const char* source, const double* t7) {
    geometry_msgs::Transform t;
    t.translation.x = t7[0];
    t.translation.y = t7[1];
    t.translation.z = t7[2];
    t.rotation.x = t7[3];
    t.rotation.y = t7[4];
    t.rotation.z = t7[5];
    t.rotation.w = t7[6];
    tf2_ros::TfTable::get().t[std::make_pair(std::string(target), std::string(source))] = t;
}

// obs rows: id, tx, ty, tz, qx, qy, qz, qw, object_error, fiducial_area.
// robot_out (optional, 14): published(0/1), t3, q4, covariance diagonal 6  -- the /fiducial_pose message of this update.
int mapref_update(void* p, int n, const double* obs, double stamp, const char* frame, double* robot_out) {
    MapRef* h = static_cast<MapRef*>(p);
    ros::Time::clock() = ros::Time(stamp);
    std::vector<Observation> observations;
    for (int i = 0; i < n; i++) {
        const double* o = obs + 10 * i;
        geometry_msgs::Transform tr;
        tr.translation.x = o[1];
        tr.translation.y = o[2];
        tr.translation.z = o[3];
        tr.rotation.x = o[4];
        tr.rotation.y = o[5];
        tr.rotation.z = o[6];
        tr.rotation.w = o[7];
        const double variance = h->use_area ? h->weighting_scale / o[9] : h->weighting_scale * o[8];
        observations.push_back(Observation((int)o[0], tf2::Stamped<TransformWithVariance>(TransformWithVariance(tr, variance), ros::Time(stamp), frame)));
    }
    const long before = ros::Capture::get().n<geometry_msgs::PoseWithCovarianceStamped>();
    h->map->update(observations, ros::Time(stamp));
    const bool published = ros::Capture::get().n<geometry_msgs::PoseWithCovarianceStamped>() > before;
    if (robot_out) {
        memset(robot_out, 0, 14 * sizeof(double));
        robot_out[0] = published ? 1.0 : 0.0;
        if (published) {
            const geometry_msgs::PoseWithCovarianceStamped* m = ros::Capture::get().peek<geometry_msgs::PoseWithCovarianceStamped>();
            robot_out[1] = m->pose.pose.position.x;
            robot_out[2] = m->pose.pose.position.y;
            robot_out[3] = m->pose.pose.position.z;
            robot_out[4] = m->pose.pose.orientation.x;
            robot_out[5] = m->pose.pose.orientation.y;
            robot_out[6] = m->pose.pose.orientation.z;
            robot_out[7] = m->pose.pose.orientation.w;
            for (int i = 0; i < 6; i++) robot_out[8 + i] = m->pose.covariance[i * 6 + i];
        }
    }
    return (int)h->map->fiducials.size();
}

// the last map -> odom / map -> base transform the Map broadcast (map.cpp:381-398): out (9) = have, t3, q4, child is odom (1) or base (0)
int mapref_pose_tf(void* p, double* out) {
    MapRef* h = static_cast<MapRef*>(p);
    out[0] = h->map->havePose ? 1.0 : 0.0;
    const geometry_msgs::TransformStamped& t = h->map->poseTf;
    out[1] = t.transform.translation.x;
    out[2] = t.transform.translation.y;
    out[3] = t.transform.translation.z;
    out[4] = t.transform.rotation.x;
    out[5] = t.transform.rotation.y;
    out[6] = t.transform.rotation.z;
    out[7] = t.transform.rotation.w;
    out[8] = t.child_frame_id == h->map->odomFrame && !h->map->odomFrame.empty() ? 1.0 : 0.0;
    return h->map->havePose ? 1 : 0;
}

// rows (10): id, x, y, z, rx, ry, rz (publishMap read-out, map.cpp:629-654), variance, numObs, n_links
int mapref_entries(void* p, int cap, double* out) {
    MapRef* h = static_cast<MapRef*>(p);
    int n = 0;
    for (const auto& kv : h->map->fiducials) {
        if (n >= cap) break;
        const Fiducial& f = kv.second;
        double* o = out + 10 * n++;
        const tf2::Vector3 t = f.pose.transform.getOrigin();
        double rx, ry, rz;
        f.pose.transform.getBasis().getRPY(rx, ry, rz);
        o[0] = f.id;
        o[1] = t.x();
        o[2] = t.y();
        o[3] = t.z();
        o[4] = rx;
        o[5] = ry;
        o[6] = rz;
        o[7] = f.pose.variance;
        o[8] = f.numObs;
        o[9] = (double)f.links.size();
    }
    return n;
}

// link pairs (id, linked id), ascending; returns the number of pairs
int mapref_links(void* p, int cap_pairs, int* out) {
    MapRef* h = static_cast<MapRef*>(p);
    int n = 0;
    for (const auto& kv : h->map->fiducials)
        for (int l : kv.second.links) {
            if (n < cap_pairs) {
                out[2 * n] = kv.first;
                out[2 * n + 1] = l;
            }
            n++;
        }
    return n;
}

void mapref_add_fiducial(void* p, int id) {
    fiducial_slam::AddFiducial::Request req;
    fiducial_slam::AddFiducial::Response res;
    req.fiducial_id = id;
    static_cast<MapRef*>(p)->map->addFiducialCallback(req, res);
}

void mapref_clear(void* p) {
    std_srvs::Empty::Request req;
    std_srvs::Empty::Response res;
    static_cast<MapRef*>(p)->map->clearCallback(req, res);
}

int mapref_load_map(void* p, const char* path) { return static_cast<MapRef*>(p)->map->loadMap(path) ? 1 : 0; }
int mapref_save_map(void* p, const char* path) { return static_cast<MapRef*>(p)->map->saveMap(path) ? 1 : 0; }

int mapref_state(void* p, int* out /* frameNum, isInitializingMap, originFid, fiducialToAdd */) {
    MapRef* h = static_cast<MapRef*>(p);
    out[0] = h->map->frameNum;
    out[1] = h->map->isInitializingMap ? 1 : 0;
    out[2] = h->map->originFid;
    out[3] = h->map->fiducialToAdd;
    return 0;
}

// Replays n_msgs messages (CSR offsets into obs rows as in mapref_update) without leaving C: the CPU arm of `bench.py --workload C5`.
int mapref_replay(void* p, int n_msgs, const int* offsets, const double* obs, double stamp0, const char* frame) {
    int n = 0;
    for (int m = 0; m < n_msgs; m++) n = mapref_update(p, offsets[m + 1] - offsets[m], obs + 10 * (size_t)offsets[m], stamp0 + 0.05 * m, frame, nullptr);
    return n;
}

// TransformWithVariance::update / operator* of the reference, directly (transform_with_variance.cpp:43-85, .h:26-59).
// a, b: x y z qx qy qz qw variance; out the same layout.  op 0: a.update(b)  1: averageTransforms(a, b)  2: a * b  3: a.inverse composed: a^-1 (variance kept)
void twvref_apply(int op, const double* a, const double* b, double* out) {
    auto mk = [](const double* v) { return TransformWithVariance(tf2::Vector3(v[0], v[1], v[2]), tf2::Quaternion(v[3], v[4], v[5], v[6]), v[7]); };
    TransformWithVariance r = mk(a);
    if (op == 0) {
        r.update(mk(b));
    } else if (op == 1) {
        r = averageTransforms(mk(a), mk(b));
    } else if (op == 2) {
        r = mk(a) * mk(b);
    } else {
        r.transform = r.transform.inverse();
    }
    const tf2::Vector3 t = r.transform.getOrigin();
    const tf2::Quaternion q = r.transform.getRotation();
    out[0] = t.x();
    out[1] = t.y();
    out[2] = t.z();
    out[3] = q.x();
    out[4] = q.y();
    out[5] = q.z();
    out[6] = q.w();
    out[7] = r.variance;
}

}  // extern "C"
