// The shim with a distorted camera, the way a reference caller would use it: PinholeCamera with k1 k2 p1 p2,
// b200::Runtime::SetUndistortion, then Frame::InitFrame and FeatureDetector::Detect on a raw frame.  Input: one raw 640x480
// grey frame followed by fx fy cx cy k1 k2 p1 p2 as float32, written by tests/test_gpu_undistort.py; prints the detected
// features, which the Python side compares with the oracle's detection on the undistorted frame.
#include <cstdio>
#include <vector>

#include "../ygz_slam_b200/host/ygz_b200.hpp"

using namespace ygz;

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    FILE* fp = fopen(argv[1], "rb");
    if (!fp) return 3;
    Frame f;
    f._color.create(480, 640, 1);
    float c[8];
    if (fread(f._color.data, 1, 640 * 480, fp) != 640 * 480 || fread(c, 4, 8, fp) != 8) return 4;
    fclose(fp);
    PinholeCamera cam(c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7]);
    Frame::SetCamera(&cam);
    b200::Runtime::Get().SetUndistortion(cam);
    f.InitFrame();
    FeatureDetector det;
    det.Detect(&f);
    printf("features %zu\n", f._features.size());
    for (const Feature* fe : f._features) {
        unsigned long long d = 0;
        for (int k = 0; k < 32; ++k) d = d * 31 + fe->_desc[k];
        printf("%.1f %.1f %d %llu\n", fe->_pixel[0], fe->_pixel[1], fe->_level, d);
    }
    return 0;
}
