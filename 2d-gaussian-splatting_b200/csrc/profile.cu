// profile.cu — launch counter + optional per-stage event timing (see profile.h).
#include <atomic>
#include <mutex>
#include <vector>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "profile.h"

namespace surfel {

namespace {
std::atomic<unsigned long long> g_launches{0};
std::atomic<int> g_enabled{0};
struct Span { int stage; cudaEvent_t a, b; };
std::mutex g_mu;
std::vector<Span> g_open[kNumStages];   // begun, not yet ended (per stage)
std::vector<Span> g_done;
std::vector<cudaEvent_t> g_pool;

cudaEvent_t get_event() {
    if (!g_pool.empty()) { cudaEvent_t e = g_pool.back(); g_pool.pop_back(); return e; }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
}  // namespace

void prof_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
bool prof_enabled() { return g_enabled.load(std::memory_order_relaxed) != 0; }

void prof_begin(int stage, cudaStream_t stream) {
    std::lock_guard<std::mutex> lk(g_mu);
    Span s{stage, get_event(), get_event()};
    cudaEventRecord(s.a, stream);
    g_open[stage].push_back(s);
}
void prof_end(int stage, cudaStream_t stream) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_open[stage].empty()) return;
    Span s = g_open[stage].back();
    g_open[stage].pop_back();
    cudaEventRecord(s.b, stream);
    g_done.push_back(s);
}

}  // namespace surfel

using namespace surfel;

extern "C" {

unsigned long long surfel_launch_count(void) { return g_launches.load(); }

void surfel_profile_enable(int on) { g_enabled.store(on ? 1 : 0); }

// Sums the recorded per-stage kernel times (ms) and launch counts since the last read, waiting for
// the events.  ms_out / count_out: arrays of surfel_profile_num_stages() entries.
int surfel_profile_num_stages(void) { return kNumStages; }
const char* surfel_profile_stage_name(int stage) {
    static const char* names[kNumStages] = {"preprocess_fwd", "duplicate_with_keys", "sort_histogram",
                                            "sort_onesweep_pass", "identify_tile_ranges", "render_fwd",
                                            "render_bwd", "preprocess_bwd", "mark_visible", "tile_count", "tile_scan",
                                            "tile_scatter", "tile_sort", "adam_step", "densify_stats", "ply_unpack", "ply_pack", "knn", "densify", "tsdf",
                                            "mcubes_crop", "mcubes_merge", "meshpost_edges", "meshpost_union",
                                            "meshpost_label", "meshpost_compact", "chamfer_sample",
                                            "chamfer_downsample", "chamfer_select", "chamfer_nn", "cull_dilate",
                                            "cull_vertices", "cull_faces", "cull_emit", "camera_bwd",
                                            "camera_finish"};
    return stage >= 0 && stage < kNumStages ? names[stage] : "";
}
int surfel_profile_read(double* ms_out, int* count_out) {
    std::lock_guard<std::mutex> lk(g_mu);
    for (int i = 0; i < kNumStages; i++) { ms_out[i] = 0.0; count_out[i] = 0; }
    for (const Span& s : g_done) {
        float ms = 0.0f;
        SURFEL_CUDA_OK(cudaEventSynchronize(s.b));
        SURFEL_CUDA_OK(cudaEventElapsedTime(&ms, s.a, s.b));
        ms_out[s.stage] += ms;
        count_out[s.stage] += 1;
        g_pool.push_back(s.a);
        g_pool.push_back(s.b);
    }
    g_done.clear();
    return 0;
}

}  // extern "C"
