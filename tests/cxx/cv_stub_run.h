// Minimal stand-ins for the OpenCV / reference types CudaCostVolumeEnergy.h touches, so that the adapter can be
// compile-checked in a container without OpenCV C++ headers.  This variant adds cv::Mat::create and CV_32FC4 for CudaCostVolumeEnergy::run.  Shapes follow cv::Mat / cv::Rect and the reference's
// StereoEnergy.h:13-40,42-118,616-626 and Plane.h:4-12; NOT a re-implementation of either.
#pragma once
#include <cstddef>
#include <string>
#include <vector>
#define CV_32FC4 29
namespace cv {
struct Rect { int x, y, width, height; };
struct MatSize { const int* p; };
struct Mat {
    unsigned char* data = nullptr;
    size_t step = 0;
    int rows = 0, cols = 0;
    int sz[3] = {0, 0, 0};
    MatSize size{sz};
    template <typename T> T* ptr() const { return reinterpret_cast<T*>(data); }
    std::vector<unsigned char> own;
    void create(int r, int c, int /*type: CV_32FC4*/) { rows = r; cols = c; step = (size_t)c * 16; own.assign((size_t)r * step, 0); data = own.data(); }
};
}  // namespace cv
struct Plane { float a, b, c, v; };
struct Parameters {
    float alpha = 0.9f, omega = 10, th_grad = 2, th_col = 10, lambda = 20, th_smooth = 1, epsilon = 0.01f, filter_param1 = 10;
    int windR = 20, neighborNum = 8;
    std::string filterName = "GF";
};
class StereoEnergy {
public:
    Parameters params;
    StereoEnergy(const cv::Mat, const cv::Mat, Parameters p, float, float = 0, float = 0) : params(p) {}
    virtual ~StereoEnergy() {}
    struct Reusable { cv::Mat pIL, pIR; cv::Rect filterRect; };
    virtual void ComputeUnaryPotentialWithoutCheck(const cv::Rect&, const cv::Rect&, const cv::Mat&, const Plane&, Reusable&, int) const {}
    virtual void ComputeUnaryPotential(const cv::Rect&, const cv::Rect&, const cv::Mat&, const Plane&, Reusable&, int) const {}
};
