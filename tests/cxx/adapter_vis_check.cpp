// Compile-and-link check of CudaCostVolumeEnergy::setSaveDir (include/CudaCostVolumeEnergy.h): run() with a save directory goes through
// lexp_run_ex and cv::imwrite, against the cv stub of cv_stub_vis.h and liblexp_cuda.so.
#define LEXP_ADAPTER_NO_REFERENCE_INCLUDES
#include "cv_stub_vis.h"
#include "../../include/CudaCostVolumeEnergy.h"
#include <cstdio>
static void on_evaluate(void*, int index, int mode, const lexp_eval_result* r, double seconds) {
    std::printf("%2d %d %5.1lf\t%.0lf\t%4.2lf\t%4.2lf\n", index, mode, seconds, r->energy, r->all, r->nonocc);
}
int main(int argc, char**) {
    std::printf("lexp version %d\n", lexp_version());
    if (argc > 100) {  // never executed: only instantiates the calls so that they are type-checked and linked
        cv::Mat im, labeling, raw;
        CudaNaiveStereoEnergy e(im, im, Parameters(), 58.f);
        e.addLayer(5, {{LEXP_PROP_EXPANSION, 1}, {LEXP_PROP_RANSAC, 1}, {LEXP_PROP_RANDOM, 7}});
        e.setRunOptions(7, 0.25f, 0.5f, on_evaluate, nullptr);
        e.setSaveDir("out/debug/");
        e.run(5, {0, 1}, 2, labeling, raw);
        e.setSaveDir("");
        e.run(5, {0}, 2, labeling, raw);
    }
    return 0;
}
