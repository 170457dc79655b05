// The stand-ins of cv_stub_run.h plus what CudaCostVolumeEnergy::setSaveDir needs: CV_8UC1 / CV_8UC3 and a cv::imwrite that writes
// nothing, so that the debug-image path of the adapter can be compile-checked without OpenCV C++ headers.
#pragma once
#include "cv_stub_run.h"
#define CV_8UC1 0
#define CV_8UC3 16
namespace cv {
inline bool imwrite(const std::string&, const Mat&) { return true; }
}  // namespace cv
