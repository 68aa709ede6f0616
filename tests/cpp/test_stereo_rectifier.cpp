// util::stereo_rectifier through adapters.hpp (the reference's constructor from the camera and the parsed StereoRectifier block,
// and rectify(const cv::Mat&, ...) on the stand-in cv::Mat) and through the class layer's array views, on the GPU.  Both must
// agree; orb_extractor::extract with the rectifier must equal extract on the rectified image.  The program writes the rig, the
// raw pair and both outputs to the directory argv[1], where tests/test_rectify_gpu.py checks them against the Python path.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "openvslam_b200/adapters.hpp"

namespace {

void write(const std::string& dir, const char* name, const void* data, std::size_t bytes) {
    FILE* f = std::fopen((dir + "/" + name + ".bin").c_str(), "wb");
    if (!f || std::fwrite(data, 1, bytes, f) != bytes) throw std::runtime_error(std::string("cannot write ") + name);
    std::fclose(f);
}

std::array<double, 9> rotation(double ax, double ay, double az) {
    const double cx = std::cos(ax), sx = std::sin(ax), cy = std::cos(ay), sy = std::sin(ay), cz = std::cos(az), sz = std::sin(az);
    // Rz Ry Rx
    return {cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx,
            sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx,
            -sy, cy * sx, cy * cx};
}

}  // namespace

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: %s out_dir\n", argv[0]); return 1; }
    const std::string dir = argv[1];
    try {
        using namespace openvslam;
        const int cols = 752, rows = 480;
        const camera::perspective cam(camera::setup_type_t::Stereo, cols, rows, 435.2, 435.2, 367.2, 252.2, 47.9);
        util::stereo_rectifier::params p;
        p.model = OVS_CAMERA_PERSPECTIVE;
        p.K_left = {458.654, 0, 367.215, 0, 457.296, 248.375, 0, 0, 1};
        p.K_right = {457.587, 0, 379.999, 0, 456.134, 255.238, 0, 0, 1};
        p.D_left = {-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0};
        p.D_right = {-0.28368365, 0.07451284, -0.00010473, -3.55590700e-05, 0.0};
        p.R_left = rotation(0.0041, -0.0093, 0.0012);
        p.R_right = rotation(0.0032, -0.0062, 0.0015);
        const util::stereo_rectifier rect(&cam, p);

        cv::Mat raw_l(rows, cols, CV_8U), raw_r(rows, cols, CV_8U);
        for (int y = 0; y < rows; ++y)
            for (int x = 0; x < cols; ++x) {
                const int v = ((x / 16 + y / 16) & 1) * 160 + (x * 7 + y * 13) % 61 + ((x * x + 3 * y) % 29);
                raw_l.ptr(y)[x] = static_cast<unsigned char>(v);
                raw_r.ptr(y)[(x + 11) % cols] = static_cast<unsigned char>(v);
            }
        cv::Mat out_l, out_r;
        rect.rectify(raw_l, raw_r, out_l, out_r);

        std::vector<std::uint8_t> cls_l(static_cast<std::size_t>(rows) * cols), cls_r(cls_l.size());
        rect.rectify(raw_l.data, raw_r.data, rows, cols, raw_l.step, 1, cls_l.data(), cls_r.data(), cols);
        for (int y = 0; y < rows; ++y)
            if (std::memcmp(out_l.ptr(y), &cls_l[static_cast<std::size_t>(y) * cols], cols) != 0 ||
                std::memcmp(out_r.ptr(y), &cls_r[static_cast<std::size_t>(y) * cols], cols) != 0) {
                std::printf("adapter and class layer differ in row %d\n", y);
                return 1;
            }

        feature::orb_extractor ext(feature::orb_params(1000, 1.2f, 8, 20, 7));
        std::vector<ovs_keypoint> k1, k2;
        std::vector<std::uint8_t> d1, d2;
        ext.extract(rect, 0, raw_l.data, rows, cols, raw_l.step, 1, OVS_COLOR_ORDER_BGR, nullptr, 0, k1, d1);
        ext.extract(cls_l.data(), rows, cols, cols, nullptr, 0, k2, d2);
        if (k1.empty() || k1.size() != k2.size() || std::memcmp(k1.data(), k2.data(), k1.size() * sizeof(ovs_keypoint)) != 0 || d1 != d2) {
            std::printf("extract with the rectifier differs from extract on the rectified image (%zu vs %zu keypoints)\n", k1.size(), k2.size());
            return 1;
        }

        std::vector<double> rig = {double(cols), double(rows)};
        const std::array<double, 9> K_rect{cam.fx_, 0, cam.cx_, 0, cam.fy_, cam.cy_, 0, 0, 1};
        for (const std::array<double, 9>* m : std::initializer_list<const std::array<double, 9>*>{&p.K_left, &p.R_left, &p.K_right, &p.R_right, &K_rect}) rig.insert(rig.end(), m->begin(), m->end());
        rig.insert(rig.end(), p.D_left.begin(), p.D_left.end());
        rig.insert(rig.end(), p.D_right.begin(), p.D_right.end());
        write(dir, "rig", rig.data(), rig.size() * sizeof(double));
        write(dir, "raw_l", raw_l.data, cls_l.size());
        write(dir, "raw_r", raw_r.data, cls_l.size());
        write(dir, "out_l", out_l.data, cls_l.size());
        write(dir, "out_r", out_r.data, cls_l.size());
        write(dir, "cls_l", cls_l.data(), cls_l.size());
        write(dir, "cls_r", cls_r.data(), cls_r.size());
        std::printf("stereo rectifier ok: %zu keypoints\n", k1.size());
        return 0;
    } catch (const std::exception& e) {
        std::printf("error: %s\n", e.what());
        return 2;
    }
}
