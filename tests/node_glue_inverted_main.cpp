// The C++ node glue with white-on-black markers (FiducialsNode::setDetectInvertedMarker): reads a raw BGR8 frame written by
// tests/test_gpu_inverted.py, runs imageCallback + poseEstimateCallback with detectInvertedMarker on, and prints the messages as text.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../fiducials_b200/csrc/node_glue.hpp"

int main(int argc, char** argv) {
    // frame.bgr width height dictionary fiducial_len
    if (argc != 6) {
        std::fprintf(stderr, "usage: %s frame.bgr width height dictionary fiducial_len\n", argv[0]);
        return 2;
    }
    const int W = std::atoi(argv[2]), H = std::atoi(argv[3]), dict = std::atoi(argv[4]);
    std::vector<uint8_t> bgr((size_t)W * H * 3);
    FILE* f = std::fopen(argv[1], "rb");
    if (!f || std::fread(bgr.data(), 1, bgr.size(), f) != bgr.size()) return 3;
    std::fclose(f);
    try {
        fid_glue::FiducialsNode node(dict, std::atof(argv[5]), W, H);
        node.setDetectInvertedMarker(true);
        double K[9] = {0.73 * W, 0, W / 2.0, 0, 0.73 * W, H / 2.0, 0, 0, 1};
        double D[5] = {-0.2, 0.05, 0.001, -0.001, 0.0};
        node.camInfoCallback(K, D, 5, "camera");
        fid_glue::FiducialArray fva;
        fid_glue::FiducialTransformArray fta;
        fid_glue::Header hdr;
        if (!node.imageCallback(bgr.data(), W, H, (size_t)W * 3, hdr, &fva)) return 4;
        if (!node.poseEstimateCallback(&fta)) return 5;
        for (const auto& v : fva.fiducials) std::printf("V %d %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g\n", v.fiducial_id, v.x0, v.y0, v.x1, v.y1, v.x2, v.y2, v.x3, v.y3);
        for (const auto& t : fta.transforms)
            std::printf("T %d %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", t.fiducial_id, t.transform.tx, t.transform.ty, t.transform.tz, t.transform.qx,
                        t.transform.qy, t.transform.qz, t.transform.qw, t.image_error, t.object_error, t.fiducial_area);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
