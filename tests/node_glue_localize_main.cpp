// The C++ node glue's localization (FiducialSlam::localize, publishedPose): reads a map file and a /fiducial_vertices message
// written by tests/test_node_glue_localize.py, localizes the frame against the map and prints the record and the published pose
// (with multi_error_theshold at -1 and at 1e9) as text.
#include <cstdio>
#include <cstdlib>
#include <fstream>

#include "../fiducials_b200/csrc/node_glue.hpp"

int main(int argc, char** argv) {
    // map.txt vertices.txt fx fy cx cy k1 k2 p1 p2 k3 fiducial_len
    if (argc != 13) {
        std::fprintf(stderr, "usage: %s map.txt vertices.txt fx fy cx cy k1 k2 p1 p2 k3 fiducial_len\n", argv[0]);
        return 2;
    }
    fid_camera cam{};
    cam.K[0] = std::atof(argv[3]);
    cam.K[4] = std::atof(argv[4]);
    cam.K[2] = std::atof(argv[5]);
    cam.K[5] = std::atof(argv[6]);
    cam.K[8] = 1.0;
    for (int k = 0; k < 5; k++) cam.D[k] = std::atof(argv[7 + k]);
    fid_glue::FiducialArray fva;
    std::ifstream in(argv[2]);
    for (fid_glue::Fiducial v; in >> v.fiducial_id >> v.x0 >> v.y0 >> v.x1 >> v.y1 >> v.x2 >> v.y2 >> v.x3 >> v.y3;) fva.fiducials.push_back(v);
    try {
        fid_glue::FiducialSlam slam(64);
        if (!slam.loadMap(argv[1])) return 3;
        const fid_tf mount{{0.12, -0.03, 0.35}, {0.5, -0.5, 0.5, 0.5}};
        const fid_localization loc = slam.localize(fva, cam, std::atof(argv[12]), {}, &mount);
        std::printf("L %d %d %d %d", loc.status, loc.n_markers, loc.start, loc.cov_ok);
        for (double v : loc.t) std::printf(" %.17g", v);
        for (double v : loc.q) std::printf(" %.17g", v);
        std::printf(" %.17g", loc.object_error);
        for (double v : loc.covariance) std::printf(" %.17g", v);
        std::printf("\n");
        const fid_robot_pose robot{1, 1, {1.0, 2.0, 0.5}, {0.0, 0.0, 0.0, 1.0}, 0.25};
        for (double thr : {-1.0, 1e9}) {
            slam.multiErrorThreshold = thr;
            double cov[36];
            const fid_glue::Transform p = slam.publishedPose(robot, &loc, cov);
            std::printf("P %.17g %.17g %.17g %.17g %.17g %.17g %.17g", p.tx, p.ty, p.tz, p.qx, p.qy, p.qz, p.qw);
            for (double v : cov) std::printf(" %.17g", v);
            std::printf("\n");
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
