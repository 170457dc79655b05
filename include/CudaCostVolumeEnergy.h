// CudaCostVolumeEnergy.h -- the reference-side binding: a StereoEnergy subclass that a maintainer of
// t-taniai/LocalExpStereo adds next to CostVolumeEnergy.h.  It keeps the virtual interface
// (StereoEnergy.h:625-626), Plane (Plane.h) and LayerManager untouched and forwards the two unary-cost
// virtuals to the C-ABI of lexp_cuda.h.  Install it exactly where the reference installs its CPU energy:
//
//     stereo.setStereoEnergyCPU(std::make_unique<CudaCostVolumeEnergy>(imL, imR, volL, volR, param, maxdisp));   // main.cpp:386
//
// Compile-checked in this repository against a minimal cv:: stub (tests/cxx/); it needs the real
// <opencv2/opencv.hpp> and StereoEnergy.h of the reference to be used for real.
#pragma once
#include "lexp_cuda.h"
#ifndef LEXP_ADAPTER_NO_REFERENCE_INCLUDES
#include "StereoEnergy.h"
#endif
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

class CudaCostVolumeEnergy : public StereoEnergy {
protected:
    lexp_ctx* ctx_ = nullptr;
    int height_ = 0, width_ = 0;
    std::vector<int> unitSizes_;                                     // addLayer / run
    std::vector<std::vector<std::pair<int, int>>> layerProposers_;
    uint64_t runSeed_ = 0;
    float runPrecision_ = -1.0f, runThreshold_ = 0.5f;
    lexp_run_callback runCallback_ = nullptr;
    void* runUser_ = nullptr;
    std::string saveDir_;                                            // setSaveDir: where run() writes the debug images

    static void check(int rc) {
        if (rc != LEXP_OK) throw std::runtime_error(std::string("lexp_cuda: ") + lexp_last_error());
    }
    static lexp_rect toRect(const cv::Rect& r) { return lexp_rect{r.x, r.y, r.width, r.height}; }

    // The two virtuals are called inside `#pragma omp parallel for` (FastGCStereo.h:30-49): an exception must not leave that
    // region (std::terminate).  A failing call records the first error, marks the whole targetRect COST_FOR_INVALID (1e6,
    // StereoEnergy.h:45 -- the fusion then never accepts the proposal there) and returns; the caller asks failed() /
    // throwIfFailed() after the parallel region (INTEGRATION.md section 2).
    mutable std::mutex err_mu_;
    mutable std::string err_;
    mutable std::atomic<bool> failed_{false};
    void guard(int rc, const cv::Rect& filterRect, const cv::Rect& targetRect, const cv::Mat& costs) const {
        if (rc == LEXP_OK) return;
        {
            std::lock_guard<std::mutex> lk(err_mu_);
            if (err_.empty()) err_ = std::string("lexp_cuda: ") + lexp_last_error();
        }
        failed_.store(true);
        for (int y = 0; y < targetRect.height; y++) {
            float* row = reinterpret_cast<float*>(costs.data + (ptrdiff_t)(targetRect.y - filterRect.y + y) * (ptrdiff_t)costs.step) + (targetRect.x - filterRect.x);
            for (int x = 0; x < targetRect.width; x++) row[x] = 1000000.0f;
        }
    }

    // shared by the two energies
    CudaCostVolumeEnergy(const cv::Mat imL, const cv::Mat imR, Parameters params, float MAX_DISPARITY, float MIN_DISPARITY, float MAX_VDISPARITY,
                         int device, int energy_kind, int ndisp)
        : StereoEnergy(imL, imR, params, MAX_DISPARITY, MIN_DISPARITY, MAX_VDISPARITY) {
        lexp_params p{};
        p.filter = filterKind(params.filterName, energy_kind);
        p.height = height_ = imL.rows; p.width = width_ = imL.cols; p.ndisp = ndisp;
        p.windR = params.windR; p.eps = params.filter_param1; p.th_col = params.th_col;
        p.min_disp = MIN_DISPARITY; p.max_disp = MAX_DISPARITY; p.device = device;
        p.energy_kind = energy_kind; p.alpha = params.alpha; p.th_grad = params.th_grad;
        check(lexp_create(&p, &ctx_));
        check(lexp_set_image(ctx_, 0, imL.data, (ptrdiff_t)imL.step));
        check(lexp_set_image(ctx_, 1, imR.data, (ptrdiff_t)imR.step));
    }

public:
    // Parameters::filterName as the reference's energies select their filter (CostVolumeEnergy.h:23-42, StereoEnergy.h:666-686).  The
    // names for which the reference leaves its filter a null pointer ("BF" with the cost-volume energy, "BL" with the image-based one,
    // anything unknown) crash it in ComputeUnaryPotential: rejected here.
    static int filterKind(const std::string& name, int energy_kind) {
        if (name == "GF" || name == "GFfloat") return LEXP_FILTER_GF;
        if (name.empty()) return LEXP_FILTER_NONE;
        if (name == (energy_kind == 0 ? "BL" : "BF")) return LEXP_FILTER_BILATERAL;
        throw std::invalid_argument(std::string("filterName \"") + name + "\": the reference's " +
                                    (energy_kind == 0 ? "CostVolumeEnergy" : "NaiveStereoEnergy") +
                                    " leaves its filter a null pointer for this name (valid: \"GF\", \"GFfloat\", \"" +
                                    (energy_kind == 0 ? "BL" : "BF") + "\", \"\")");
    }

    // same argument list as CostVolumeEnergy::CostVolumeEnergy (CostVolumeEnergy.h:16)
    CudaCostVolumeEnergy(const cv::Mat imL, const cv::Mat imR, const cv::Mat volL, const cv::Mat volR, Parameters params,
                         float MAX_DISPARITY, float MIN_DISPARITY = 0, float MAX_VDISPARITY = 0, int device = 0)
        : CudaCostVolumeEnergy(imL, imR, params, MAX_DISPARITY, MIN_DISPARITY, MAX_VDISPARITY, device, 0, volL.size.p[0]) {
        check(lexp_set_volume_host(ctx_, 0, volL.ptr<float>()));   // float[D][H][W], continuous (main.cpp:353-354)
        check(lexp_set_volume_host(ctx_, 1, volR.ptr<float>()));
    }
    // The cost volumes straight from the reference's files (main.cpp:353-370: `im0.acrt`, raw float[ndisp][H][W]), streamed in slabs with
    // fillOutOfView fused in; without `im1.acrt` the right volume is derived from the left file (convertVolumeL2R + both fills, :363-367).
    // Replaces `loadMatBinary + fillOutOfView (+ convertVolumeL2R)` and the 2 x 17 GB of host memory they need at 4K.
    CudaCostVolumeEnergy(const cv::Mat imL, const cv::Mat imR, const std::string& volLFile, const std::string& volRFileOrEmpty, int ndisp,
                         Parameters params, float MAX_DISPARITY, float MIN_DISPARITY = 0, float MAX_VDISPARITY = 0, int device = 0)
        : CudaCostVolumeEnergy(imL, imR, params, MAX_DISPARITY, MIN_DISPARITY, MAX_VDISPARITY, device, 0, ndisp) {
        check(lexp_set_volume_file(ctx_, 0, volLFile.c_str(), LEXP_VOL_FILL));
        if (volRFileOrEmpty.empty()) check(lexp_set_volume_file(ctx_, 1, volLFile.c_str(), LEXP_VOL_RIGHT_FROM_LEFT));
        else check(lexp_set_volume_file(ctx_, 1, volRFileOrEmpty.c_str(), LEXP_VOL_FILL));
    }
    ~CudaCostVolumeEnergy() override { lexp_destroy(ctx_); }
    CudaCostVolumeEnergy(const CudaCostVolumeEnergy&) = delete;
    CudaCostVolumeEnergy& operator=(const CudaCostVolumeEnergy&) = delete;

    // `costs` is proposalCost(filterRect) (FastGCStereo.h:49): costs.data addresses element (filterRect.y, filterRect.x).
    // `reusable` is unused: the per-cell sub-filter it caches on the CPU (GuidedFilter.h:301-326) has no device state.
    void ComputeUnaryPotentialWithoutCheck(const cv::Rect& filterRect, const cv::Rect& targetRect, const cv::Mat& costs,
                                           const Plane& plane, Reusable& reusable = defaultReusable(), int mode = 0) const override {
        (void)reusable;
        const lexp_rect f = toRect(filterRect), t = toRect(targetRect);
        const lexp_plane pl{plane.a, plane.b, plane.c, plane.v};
        guard(lexp_eval_cell(ctx_, mode, &f, &t, &pl, reinterpret_cast<float*>(costs.data), (ptrdiff_t)costs.step, 0), filterRect, targetRect, costs);
    }
    void ComputeUnaryPotential(const cv::Rect& filterRect, const cv::Rect& targetRect, const cv::Mat& costs, const Plane& plane,
                               Reusable& reusable = defaultReusable(), int mode = 0) const override {
        (void)reusable;
        const lexp_rect f = toRect(filterRect), t = toRect(targetRect);
        const lexp_plane pl{plane.a, plane.b, plane.c, plane.v};
        guard(lexp_eval_cell(ctx_, mode, &f, &t, &pl, reinterpret_cast<float*>(costs.data), (ptrdiff_t)costs.step, 1), filterRect, targetRect, costs);
    }

    // Batched form for a loop that has been restructured step-wise (INTEGRATION.md section 3): one call per
    // (layer, group, proposal step) instead of one per cell; proposalCost is the full H x W image (FastGCStereo.h:25).
    void ComputeUnaryPotentialBatch(const std::vector<cv::Rect>& filterRects, const std::vector<cv::Rect>& targetRects,
                                    cv::Mat& proposalCost, const std::vector<Plane>& planes, int mode = 0, bool check_valid = true) const {
        std::vector<lexp_rect> f(filterRects.size()), t(targetRects.size());
        for (size_t i = 0; i < f.size(); i++) { f[i] = toRect(filterRects[i]); t[i] = toRect(targetRects[i]); }
        static_assert(sizeof(Plane) == sizeof(lexp_plane), "Plane must stay {a,b,c,v} floats (Plane.h:4-8)");
        check(lexp_eval_batch(ctx_, mode, (int)f.size(), f.data(), t.data(), reinterpret_cast<const lexp_plane*>(planes.data()),
                              reinterpret_cast<float*>(proposalCost.data), (ptrdiff_t)proposalCost.step, check_valid ? 1 : 0));
    }

    // PMStereoBase::postProcess(currentLabeling_[0], currentLabeling_[1], threshold) (PMStereoBase.h:146-256) on the device state of both
    // views (PatchMatchPhase for each), in place: the tail of a two-view run (INTEGRATION.md section 4c).  Needs lexp_set_smoothness (omega).
    void postProcess(float threshold = 1.5f) const { check(lexp_post_process(ctx_, threshold, nullptr)); }

    // FastGCStereo::addLayer(unitRegionSize, proposers) and FastGCStereo::run(maxIteration, viewModes, pmInit, labeling, rawlabeling)
    // (FastGCStereo.h:86-92,133-222) in one device call (lexp_run, INTEGRATION.md section 4d).  Proposers as (LEXP_PROP_*, K) pairs.
    // An empty `labeling` starts from random labels; a given H x W CV_32FC4 labeling is the start of every view.  On return `labeling` /
    // `rawlabeling` hold view 0 after / before the post-processing (H x W CV_32FC4).  setRunOptions: the run seed (the reference seeds
    // cv::theRNG() from the clock) and the Evaluator's precision / threshold with a callback at its points (lexp_set_ground_truth first).
    // setSaveDir(dir): as `stereo.saveDir = outputDir + "debug\\"` with the Evaluator's saveDir (main.cpp:291-297): run() then writes the
    // reference's debug images with cv::imwrite -- dir + "result{m}{D,N,E}{ii}.png" at every evaluation point and, with two views,
    // dir + "result{0,1}C{ii}.png" after every iteration and the post-processing (lexp_run_ex, DESIGN.md 3j; needs lexp_set_ground_truth).
    // An empty dir (the default) writes none.  setSaveDir exists where the cv:: layer has cv::imwrite and CV_8UC1 / CV_8UC3 (OpenCV does).
    void addLayer(int unitRegionSize, const std::vector<std::pair<int, int>>& proposers) {
        unitSizes_.push_back(unitRegionSize);
        layerProposers_.push_back(proposers);
    }
    void setRunOptions(uint64_t seed, float precision = -1.0f, float threshold = 0.5f, lexp_run_callback callback = nullptr, void* user = nullptr) {
        runSeed_ = seed; runPrecision_ = precision; runThreshold_ = threshold; runCallback_ = callback; runUser_ = user;
    }
#ifdef CV_32FC4   // OpenCV's Mat::create / CV_32FC4 (a cv:: stand-in without them leaves run out)
#ifdef CV_8UC3    // and cv::imwrite of 8-bit images (a stand-in without CV_8UC3 leaves the debug images out)
    void setSaveDir(const std::string& dir) { saveDir_ = dir; }
#endif
    void run(int maxIteration, const std::vector<int>& viewModes, int pmInit, cv::Mat& labeling, cv::Mat& rawlabeling) const {
        const bool dual = viewModes.size() == 2 && viewModes[0] == 0 && viewModes[1] == 1;
        if (!dual && !(viewModes.size() == 1 && viewModes[0] == 0)) throw std::invalid_argument("run: viewModes must be {0} or {0, 1}");
        std::vector<int> np, kind, K;
        for (const auto& pl : layerProposers_) {
            np.push_back((int)pl.size());
            for (const auto& p : pl) { kind.push_back(p.first); K.push_back(p.second); }
        }
        const bool given = labeling.data != nullptr;
        if (given && (labeling.rows != height_ || labeling.cols != width_ || labeling.step != (size_t)width_ * sizeof(lexp_plane)))
            throw std::invalid_argument("run: the given labeling must be a continuous H x W CV_32FC4 mat");
        std::vector<lexp_plane> lab((size_t)height_ * width_), raw((size_t)height_ * width_);
        lexp_run_options o{dual ? 2 : 1, pmInit, maxIteration, (int)unitSizes_.size(), unitSizes_.data(), np.data(), kind.data(), K.data(),
                           given ? reinterpret_cast<const lexp_plane*>(labeling.data) : nullptr, runSeed_, runPrecision_, runThreshold_};
#ifdef CV_8UC3
        if (!saveDir_.empty()) {
            RunUser u{this, runUser_, false, std::string()};
            const int rc = lexp_run_ex(ctx_, &o, lab.data(), raw.data(), runCallback_ ? forwardEvaluation : nullptr, writeImage, &u);
            if (u.writeFailed) throw std::runtime_error("run: cv::imwrite failed for " + u.failedPath);
            check(rc);
        } else
#endif
            check(lexp_run(ctx_, &o, lab.data(), raw.data(), runCallback_, runUser_));
        labeling.create(height_, width_, CV_32FC4);
        rawlabeling.create(height_, width_, CV_32FC4);
        for (int y = 0; y < height_; y++) {
            std::memcpy(labeling.data + labeling.step * (size_t)y, &lab[(size_t)y * width_], (size_t)width_ * sizeof(lexp_plane));
            std::memcpy(rawlabeling.data + rawlabeling.step * (size_t)y, &raw[(size_t)y * width_], (size_t)width_ * sizeof(lexp_plane));
        }
    }

#ifdef CV_8UC3
private:
    struct RunUser { const CudaCostVolumeEnergy* self; void* user; bool writeFailed; std::string failedPath; };
    static void forwardEvaluation(void* u, int index, int mode, const lexp_eval_result* r, double seconds) {
        const RunUser* ru = static_cast<const RunUser*>(u);
        ru->self->runCallback_(ru->user, index, mode, r, seconds);
    }
    // Evaluator.h:164-166 (header "result") and FastGCStereo.h:164-165: one 8-bit image of lexp_run_ex, copied into a cv::Mat
    static void writeImage(void* u, int index, int mode, int kind, const uint8_t* pixels, int width, int height, int channels) {
        RunUser* ru = static_cast<RunUser*>(u);
        if (ru->writeFailed) return;
        cv::Mat m;
        m.create(height, width, channels == 1 ? CV_8UC1 : CV_8UC3);
        for (int y = 0; y < height; y++) std::memcpy(m.data + m.step * (size_t)y, pixels + (size_t)y * width * channels, (size_t)width * channels);
        char name[64];
        std::snprintf(name, sizeof name, "result%d%c%02d.png", mode, "DNEC"[kind], index);
        const std::string path = ru->self->saveDir_ + name;
        if (!cv::imwrite(path, m)) { ru->writeFailed = true; ru->failedPath = path; }
    }

public:
#endif
#endif

    lexp_ctx* context() const { return ctx_; }
    // error state of the per-cell virtuals (they never throw, see guard()): check after the OpenMP region
    bool failed() const { return failed_.load(); }
    void throwIfFailed() const {
        if (!failed_.load()) return;
        std::lock_guard<std::mutex> lk(err_mu_);
        throw std::runtime_error(err_);
    }

    // The cells of one disjoint group with their work list resident on the device.  Build it once per (layer, group) -- the
    // rectangles never change (LayerManager.h:14-24) -- and evaluate it once per proposal step: this is the fast path of
    // INTEGRATION.md section 3 (one launch for all cells of the group instead of one call per cell).
    class GroupPlan {
        lexp_ctx* ctx_;
        lexp_plan* plan_ = nullptr;
        std::vector<cv::Rect> targets_;
        std::vector<size_t> offsets_;  // float offset of cell i's tile: sum of the targetRect areas of cells 0..i-1
        size_t total_ = 0;

    public:
        GroupPlan(const CudaCostVolumeEnergy& e, const std::vector<cv::Rect>& filterRects, const std::vector<cv::Rect>& targetRects)
            : ctx_(e.context()), targets_(targetRects), offsets_(targetRects.size()) {
            if (filterRects.size() != targetRects.size()) throw std::invalid_argument("GroupPlan: one filterRect per targetRect");
            std::vector<lexp_rect> f(filterRects.size()), t(targetRects.size());
            for (size_t i = 0; i < f.size(); i++) {
                f[i] = toRect(filterRects[i]); t[i] = toRect(targetRects[i]);
                offsets_[i] = total_;
                total_ += (size_t)targetRects[i].width * targetRects[i].height;
            }
            check(lexp_plan_create(ctx_, (int)f.size(), f.data(), t.data(), &plan_));
        }
        ~GroupPlan() { lexp_plan_destroy(plan_); }
        GroupPlan(const GroupPlan&) = delete;
        GroupPlan& operator=(const GroupPlan&) = delete;

        size_t cells() const { return targets_.size(); }
        size_t tileFloats() const { return total_; }
        size_t tileOffset(size_t i) const { return offsets_[i]; }

        // one proposal step: the costs of planes[i] for cell i go to proposalCost(targetRects[i]) of the H x W image
        // (FastGCStereo.h:25,49); host memory, blocking; zero-copy if the image was registered with lexp_host_register
        void evaluate(const std::vector<Plane>& planes, cv::Mat& proposalCost, int mode = 0, bool check_valid = true) const {
            if (planes.size() != targets_.size()) throw std::invalid_argument("GroupPlan: one plane per cell");
            static_assert(sizeof(Plane) == sizeof(lexp_plane), "Plane must stay {a,b,c,v} floats (Plane.h:4-8)");
            check(lexp_plan_eval_host(ctx_, plan_, mode, reinterpret_cast<const lexp_plane*>(planes.data()),
                                      reinterpret_cast<float*>(proposalCost.data), (ptrdiff_t)proposalCost.step, check_valid ? 1 : 0));
        }
        // the same costs as contiguous tiles: cell i at tiles + tileOffset(i), row pitch targetRects[i].width
        void evaluateTiles(const std::vector<Plane>& planes, float* tiles, int mode = 0, bool check_valid = true) const {
            if (planes.size() != targets_.size()) throw std::invalid_argument("GroupPlan: one plane per cell");
            check(lexp_plan_eval_host_tiles(ctx_, plan_, mode, reinterpret_cast<const lexp_plane*>(planes.data()), tiles, check_valid ? 1 : 0));
        }
#ifndef LEXP_ADAPTER_NO_REFERENCE_INCLUDES
        // cv::Mat header over cell i's tile: what the fusion step reads as `subProposalCost` (FastGCStereo.h:37,52-58)
        cv::Mat tile(float* tiles, size_t i) const { return cv::Mat(targets_[i].height, targets_[i].width, CV_32F, tiles + offsets_[i]); }
#endif
    };

    // The PatchMatch phase of FastGCStereo::run on the device: `for (iteration < pmInit) for (layers) localExpansionMovesForLayer_CPU(...,
    // doGC = false)` (FastGCStereo.h:143-157) and initCurrentFast (:94-131), with currentCost_ / currentLabeling_ resident in HBM, the
    // proposals of ExpansionProposer / RandomProposer / RansacProposer(1) drawn on the device and the `cur > prop` update fused into the
    // unary-cost kernel.  graphCutIteration takes the same lists.
    // A maintainer replaces the pm loop of run() by (INTEGRATION.md section 4):
    //     CudaCostVolumeEnergy::PatchMatchPhase pm(energy, mode, {5, 15, 25}, {{{LEXP_PROP_EXPANSION, 1}, {LEXP_PROP_RANSAC, 1}, {LEXP_PROP_RANDOM, 7}}, ...});
    //     pm.begin(); pm.init(labels); for (it < pmInit) pm.iteration(it, seed); pm.get(currentCost_[mode], currentLabeling_[mode]);
    // Both energies: with CudaNaiveStereoEnergy (`-mode MiddV2`, single GPU) the whole run of main.cpp:310-312 is begin, init,
    // iteration x 2 (pmIterations), graphCutIteration x 5, disparities, savePfm.
    class PatchMatchPhase {
        lexp_ctx* ctx_;
        lexp_pm_sweep* sweep_ = nullptr;
        int mode_;

    public:
        typedef std::vector<std::pair<int, int>> ProposerList;   // (LEXP_PROP_EXPANSION | LEXP_PROP_RANDOM | LEXP_PROP_RANSAC, K) in the order of
                                                                 // layer.proposers; LEXP_PROP_RANSAC with K = 1 and world = 1 only
        PatchMatchPhase(const CudaCostVolumeEnergy& e, int mode, const std::vector<int>& unitSizes, const std::vector<ProposerList>& proposers,
                        int rank = 0, int world = 1)
            : ctx_(e.context()), mode_(mode) {
            if (unitSizes.size() != proposers.size()) throw std::invalid_argument("PatchMatchPhase: one proposer list per layer");
            std::vector<int> np, kind, K;
            for (const ProposerList& pl : proposers) {
                np.push_back((int)pl.size());
                for (const auto& p : pl) { kind.push_back(p.first); K.push_back(p.second); }
            }
            check(lexp_pm_sweep_create(ctx_, mode, (int)unitSizes.size(), unitSizes.data(), np.data(), kind.data(), K.data(), rank, world, &sweep_));
        }
        ~PatchMatchPhase() { lexp_pm_sweep_destroy(sweep_); }
        PatchMatchPhase(const PatchMatchPhase&) = delete;
        PatchMatchPhase& operator=(const PatchMatchPhase&) = delete;

        // currentCost_[mode] = INFINITY, currentLabeling_[mode] = 0 (FastGCStereo.h:137), or the caller's H x W mats (CV_32F / CV_32FC4, continuous)
        void begin() { check(lexp_pm_begin(ctx_, mode_, nullptr, nullptr)); }
        void begin(const cv::Mat& currentCost, const cv::Mat& currentLabeling) {
            static_assert(sizeof(Plane) == sizeof(lexp_plane), "Plane must stay {a,b,c,v} floats (Plane.h:4-8)");
            check(lexp_pm_begin(ctx_, mode_, reinterpret_cast<const float*>(currentCost.data), reinterpret_cast<const lexp_plane*>(currentLabeling.data)));
        }
        int numInitLabels() const { return lexp_pm_sweep_num_init_labels(sweep_); }
        // initCurrentFast (:101-113): labels[j] = createRandomLabel(random pixel of unitRegions[j]) of layer 0, drawn by the caller
        void init(const std::vector<Plane>& labels) {
            if ((int)labels.size() != numInitLabels()) throw std::invalid_argument("PatchMatchPhase: one label per unit region of layer 0");
            check(lexp_pm_sweep_init(sweep_, reinterpret_cast<const lexp_plane*>(labels.data())));
        }
        // initCurrentFast started from a given labeling (FastGCStereo.h:116-130): currentLabeling_[mode] = labeling (H x W CV_32FC4,
        // continuous) and, for every pixel p, currentCost_[mode](p) = ComputeUnaryPotential((p - windR, 2 windR + 1) & image, {p}, .,
        // labeling(p)) -- one launch on the device instead of one blocking call per pixel.  Resumes or warm-starts a run.
        // After postProcess, which changes the labels but not the costs, lexp_pm_init_from_labeling(ctx, mode) on each view recomputes
        // currentCost_ for the post-processed labeling (then lexp_energy reports the data term of the final state).
        void initFromLabeling(const cv::Mat& labeling) {
            static_assert(sizeof(Plane) == sizeof(lexp_plane), "Plane must stay {a,b,c,v} floats (Plane.h:4-8)");
            check(lexp_pm_begin(ctx_, mode_, nullptr, reinterpret_cast<const lexp_plane*>(labeling.data)));
            check(lexp_pm_init_from_labeling(ctx_, mode_));
        }
        int iteration(int iteration, uint64_t seed) {
            int n = 0;
            check(lexp_pm_sweep_iteration(sweep_, iteration, seed, &n));
            return n;
        }
        // One iteration of the MAIN loop of FastGCStereo::run (FastGCStereo.h:171-184: localExpansionMovesForLayer_CPU with doGC == true)
        // on the same device state: per proposal step the proposals, ComputeUnaryPotential, the pairwise terms
        // (computeSmoothnessTermsExpansion), the graph of expansionMoveBK and its minimum cut, and the copyTo / setTo of the winners
        // (FastGCStereo.h:47-59, 411-597) all run on the device.  The smoothness parameters are the energy's `params` (lambda, omega,
        // th_smooth, epsilon: StereoEnergy.h:26-36), handed over by CudaCostVolumeEnergy::setSmoothness.  Single GPU.
        int graphCutIteration(int iteration, uint64_t seed) {
            int n = 0;
            check(lexp_pm_sweep_gc_iteration(sweep_, iteration, seed, &n));
            return n;
        }
        // computeDisparities(currentLabeling_[mode]) of the device state (StereoEnergy.h:269-272) into a continuous H x W CV_32F mat, and
        // the PFM file main.cpp:319,410 writes from it (cvutils::io::save_pfm_file, byte-identical)
        void disparities(cv::Mat& disp) const { check(lexp_get_disparities(ctx_, mode_, reinterpret_cast<float*>(disp.data))); }
        static void savePfm(const std::string& file, const cv::Mat& disp) {
            check(lexp_save_pfm(file.c_str(), reinterpret_cast<const float*>(disp.data), disp.cols, disp.rows, (ptrdiff_t)disp.step));
        }
        // data term (sum of currentCost_) and StereoEnergy::computeSmoothnessCost of the device state (what the reference's Evaluator logs)
        void energy(double& dataTerm, double& smoothnessTerm) const { check(lexp_energy(ctx_, mode_, &dataTerm, &smoothnessTerm)); }
        // blocking: the state back into the caller's continuous H x W mats
        void get(cv::Mat& currentCost, cv::Mat& currentLabeling) const {
            check(lexp_pm_get(ctx_, mode_, reinterpret_cast<float*>(currentCost.data), reinterpret_cast<lexp_plane*>(currentLabeling.data)));
        }
    };

    // Parameters::lambda / omega / th_smooth / epsilon of the pairwise term (StereoEnergy.h:26-36, main.cpp:286,350) for the device-side
    // graph-cut iterations; the coefficient maps of initSmoothnessCoeff (StereoEnergy.h:131-163) are rebuilt on the device.
    void setSmoothness(const Parameters& p) { check(lexp_set_smoothness(ctx_, p.lambda, p.omega, p.th_smooth, p.epsilon)); }

private:
    // The reference declares `Reusable& reusable = Reusable()` (an MSVC extension binding a temporary to a non-const
    // reference); a conforming compiler needs an lvalue.
    static Reusable& defaultReusable() {
        static thread_local Reusable r;
        return r;
    }
};

// NaiveStereoEnergy (StereoEnergy.h:629-764) on the device: the image-based unary term of `-mode MiddV2`.  The reference builds it
// inside the PMStereoBase constructor (PMStereoBase.h:37); replace it the same way as above:
//     stereo.setStereoEnergyCPU(std::make_unique<CudaNaiveStereoEnergy>(imL, imR, param, maxdisp));
// or run the demo's whole optimisation on the device (main.cpp:310-312, INTEGRATION.md section 4b) with a PatchMatchPhase on it, layers
// {5, 15, 25}: begin, init, iteration x 2, graphCutIteration x 5, disparities, savePfm.
class CudaNaiveStereoEnergy : public CudaCostVolumeEnergy {
public:
    CudaNaiveStereoEnergy(const cv::Mat imL, const cv::Mat imR, Parameters params, float MAX_DISPARITY, float MIN_DISPARITY = 0,
                          float MAX_VDISPARITY = 0, int device = 0)
        : CudaCostVolumeEnergy(imL, imR, params, MAX_DISPARITY, MIN_DISPARITY, MAX_VDISPARITY, device, 1, (int)MAX_DISPARITY + 1) {}
};
