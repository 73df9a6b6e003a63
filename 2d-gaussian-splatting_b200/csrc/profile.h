// profile.h — launch counter and optional per-stage CUDA-event timing (used by bench.py to report
// the dominant kernel's live duration and the number of kernels launched per step).
#pragma once
#include <cuda_runtime.h>

namespace surfel {

enum Stage { kStPreFwd = 0, kStDuplicate, kStSortHist, kStSortPass, kStRanges, kStRenderFwd,
             kStRenderBwd, kStPreBwd, kStMarkVisible, kStTileCount, kStTileScan, kStTileScatter,
             kStTileSort, kStAdam, kStDensifyStats, kStPlyUnpack, kStPlyPack, kStKnn, kStDensify, kStTsdf, kStMcubesCrop,
             kStMcubesMerge, kStMeshpostEdges, kStMeshpostUnion, kStMeshpostLabel, kStMeshpostCompact,
             kStChamferSample, kStChamferDownsample, kStChamferSelect, kStChamferNn,
             kStCullDilate, kStCullVertices, kStCullFaces, kStCullEmit, kStCameraBwd, kStCameraFinish, kNumStages };

void prof_count_launch();
bool prof_enabled();
void prof_begin(int stage, cudaStream_t stream);
void prof_end(int stage, cudaStream_t stream);

// RAII: counts one kernel launch; when profiling is on, brackets it with events on `stream`.
struct LaunchScope {
    int stage; cudaStream_t stream; bool on;
    LaunchScope(int st, cudaStream_t s) : stage(st), stream(s), on(prof_enabled()) {
        prof_count_launch();
        if (on) prof_begin(stage, stream);
    }
    ~LaunchScope() { if (on) prof_end(stage, stream); }
};

}  // namespace surfel
