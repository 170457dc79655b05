// The adapter's filterName mapping (include/CudaCostVolumeEnergy.h) against the cv stub: the names the reference leaves a null filter
// for throw std::invalid_argument before any device call; the names it maps to a filter reach lexp_create (which then refuses the
// stub's empty image with a runtime_error).
#define LEXP_ADAPTER_NO_REFERENCE_INCLUDES
#include "cv_stub.h"
#include "../../include/CudaCostVolumeEnergy.h"
#include <cstdio>

template <class Make>
static int outcome(Make make) {   // 0: invalid_argument, 1: runtime_error, 2: constructed
    try { make(); } catch (const std::invalid_argument&) { return 0; } catch (const std::runtime_error&) { return 1; }
    return 2;
}

int main() {
    cv::Mat im, vol;
    int bad = 0;
    auto cv_energy = [&](const char* name) { Parameters p; p.filterName = name; return outcome([&] { CudaCostVolumeEnergy e(im, im, vol, vol, p, 63.f); }); };
    auto naive = [&](const char* name) { Parameters p; p.filterName = name; return outcome([&] { CudaNaiveStereoEnergy e(im, im, p, 63.f); }); };
    for (const char* n : {"GF", "GFfloat", "BL", ""}) if (cv_energy(n) != 1) { std::printf("CostVolumeEnergy \"%s\" not accepted\n", n); bad++; }
    for (const char* n : {"BF", "gf", "median"}) if (cv_energy(n) != 0) { std::printf("CostVolumeEnergy \"%s\" not rejected\n", n); bad++; }
    for (const char* n : {"GF", "GFfloat", "BF", ""}) if (naive(n) != 1) { std::printf("NaiveStereoEnergy \"%s\" not accepted\n", n); bad++; }
    for (const char* n : {"BL", "bf"}) if (naive(n) != 0) { std::printf("NaiveStereoEnergy \"%s\" not rejected\n", n); bad++; }
    // the filter each accepted name selects (lexp_params.filter)
    const struct { const char* name; int kind, want; } maps[] = {
        {"GF", 0, LEXP_FILTER_GF}, {"GFfloat", 0, LEXP_FILTER_GF}, {"BL", 0, LEXP_FILTER_BILATERAL}, {"", 0, LEXP_FILTER_NONE},
        {"GF", 1, LEXP_FILTER_GF}, {"GFfloat", 1, LEXP_FILTER_GF}, {"BF", 1, LEXP_FILTER_BILATERAL}, {"", 1, LEXP_FILTER_NONE}};
    for (const auto& m : maps)
        if (CudaCostVolumeEnergy::filterKind(m.name, m.kind) != m.want) { std::printf("\"%s\" (energy %d) maps to the wrong filter\n", m.name, m.kind); bad++; }
    std::printf(bad ? "FAILED\n" : "filter names ok\n");
    return bad ? 1 : 0;
}
