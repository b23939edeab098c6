// abi.cu -- the extern "C" boundary declared in include/splatam_b200.h: argument checks, workspace
// carving, stage sequencing.  No torch, no STL types in any signature.
#include "common.cuh"
#include "radix_sort.cuh"
#include <string.h>
#include <stdio.h>
#include <vector>

namespace sb {

static thread_local char g_cuda_error[512] = "";

void set_cuda_error(cudaError_t e, const char* where) {
    snprintf(g_cuda_error, sizeof(g_cuda_error), "%s: %s (%s)", where, cudaGetErrorName(e), cudaGetErrorString(e));
}

// ---- stage profiler ----
struct StageRec { int stage; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::vector<StageRec> g_prof;
ScopedStage::ScopedStage(int stage, cudaStream_t s) : slot(-1), st(s) {
    if (!g_prof_on) return;
    StageRec r; r.stage = stage;
    if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
    cudaEventRecord(r.a, st);
    g_prof.push_back(r);
    slot = (int)g_prof.size() - 1;
}
ScopedStage::~ScopedStage() { if (slot >= 0) cudaEventRecord(g_prof[slot].b, st); }

GeometryWs carve_geometry(void* ws, int P, size_t* total) {
    Carver c(ws);
    GeometryWs g;
    const size_t n = (size_t)(P > 0 ? P : 1);
    g.header = c.take<int32_t>(64);
    g.depth_key = c.take<uint32_t>(n);
    g.tiles_touched = c.take<uint32_t>(n);
    g.geom = c.take<float4>(2 * n);
    g.rect = c.take<uint2>(n);
    g.sorted_key = c.take<uint32_t>(n);
    g.sorted_idx = c.take<uint32_t>(n);
    g.offsets = c.take<uint32_t>(n);
    g.sort_temp_bytes = radix_temp_bytes((int)n, 32);
    g.sort_temp = c.take<char>(g.sort_temp_bytes);
    g.scan_temp_bytes = geometry_scan_temp_bytes((int)n);
    g.scan_temp = c.take<char>(g.scan_temp_bytes);
    if (total) *total = c.used();
    return g;
}

BinningWs carve_binning(void* ws, int R, int tiles, int color_sets, size_t* total) {
    Carver c(ws);
    BinningWs b;
    const size_t n = (size_t)(R > 0 ? R : 1);
    b.tile_unsorted = c.take<uint32_t>(n);
    b.val_unsorted = c.take<uint32_t>(n);
    b.tile_sorted = c.take<uint32_t>(n);
    b.point_list = c.take<uint32_t>(n);
    b.recA = c.take<float4>(n);
    b.recB = c.take<float4>(n);
    b.recC = c.take<float4>(n);
    b.sort_temp_bytes = radix_temp_bytes((int)n, (int)higher_msb((uint32_t)tiles));
    b.sort_temp = c.take<char>(b.sort_temp_bytes);
    b.recD = color_sets > 1 ? c.take<float4>(n) : nullptr;   // after everything else: the 1-set layout is a prefix
    if (total) *total = c.used();
    return b;
}

ImageWs carve_image(void* ws, int W, int H, size_t* total) {
    Carver c(ws);
    ImageWs img;
    const size_t tiles = (size_t)((W + kTile - 1) / kTile) * ((H + kTile - 1) / kTile);
    img.ranges = c.take<uint2>(tiles);
    img.final_T = c.take<float>((size_t)W * H);
    img.n_contrib = c.take<uint32_t>((size_t)W * H);
    if (total) *total = c.used();
    return img;
}

static bool settings_ok(const sb_settings* s) {
    return s && s->image_width > 0 && s->image_height > 0 && s->bg && s->viewmatrix && s->projmatrix &&
           (s->image_width + kTile - 1) / kTile <= 65535 && (s->image_height + kTile - 1) / kTile <= 65535;
}
static int tiles_of(const sb_settings* s) {
    return ((s->image_width + kTile - 1) / kTile) * ((s->image_height + kTile - 1) / kTile);
}

// Small helper kernels for the inspection entry points.
__global__ void export_geometry_kernel(int P, const uint32_t* depth_key, const float4* geom,
                                       const uint32_t* tiles_touched, float* depths, float* means2D,
                                       float* conic_opacity, uint32_t* tt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const uint32_t n = tiles_touched[i];
    const bool vis = n != 0u;
    if (depths) depths[i] = vis ? __uint_as_float(depth_key[i]) : 0.f;
    if (means2D) { means2D[2 * i] = vis ? geom[2 * i].x : 0.f; means2D[2 * i + 1] = vis ? geom[2 * i].y : 0.f; }
    if (conic_opacity)
        reinterpret_cast<float4*>(conic_opacity)[i] = vis ? geom[2 * i + 1] : make_float4(0.f, 0.f, 0.f, 0.f);
    if (tt) tt[i] = n;
}
template <typename KeyT>
__global__ void export_keys_kernel(int R, const KeyT* tile_sorted, const uint32_t* point_list,
                                   const uint32_t* depth_key, uint64_t* keys, uint32_t* list) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R) return;
    const uint32_t g = point_list[i];
    if (keys) keys[i] = ((uint64_t)tile_sorted[i] << 32) | (uint64_t)depth_key[g];
    if (list) list[i] = g;
}
__global__ void export_cover_kernel(int R, const float4* recA, uint8_t* cover) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R) cover[i] = (uint8_t)__float_as_uint(recA[i].z);
}

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_abi_version(void) { return SB_ABI_VERSION; }

SB_API const char* sb_status_string(int status) {
    switch (status) {
        case SB_OK: return "SB_OK";
        case SB_ERR_BAD_ARG: return "SB_ERR_BAD_ARG";
        case SB_ERR_WORKSPACE: return "SB_ERR_WORKSPACE";
        case SB_ERR_CUDA: return "SB_ERR_CUDA";
        case SB_ERR_UNSUPPORTED: return "SB_ERR_UNSUPPORTED";
        case SB_ERR_BINNING_TOO_SMALL: return "SB_ERR_BINNING_TOO_SMALL";
        default: return "SB_ERR_UNKNOWN";
    }
}

SB_API const char* sb_last_cuda_error(void) { return g_cuda_error; }

SB_API int sb_geometry_workspace_bytes(int P, size_t* bytes) {
    if (P < 0 || !bytes) return SB_ERR_BAD_ARG;
    carve_geometry(nullptr, P, bytes);
    return SB_OK;
}
SB_API int sb_image_workspace_bytes(int width, int height, size_t* bytes) {
    if (width <= 0 || height <= 0 || !bytes) return SB_ERR_BAD_ARG;
    carve_image(nullptr, width, height, bytes);
    return SB_OK;
}
SB_API int sb_binning_workspace_bytes(int num_rendered, int width, int height, int color_sets, size_t* bytes) {
    if (num_rendered < 0 || width <= 0 || height <= 0 || !bytes || color_sets < 1 || color_sets > 2) return SB_ERR_BAD_ARG;
    const int tiles = ((width + kTile - 1) / kTile) * ((height + kTile - 1) / kTile);
    carve_binning(nullptr, num_rendered, tiles, color_sets, bytes);
    return SB_OK;
}
SB_API int sb_backward_workspace_bytes(int P, int color_sets, size_t* bytes) {
    if (P < 0 || !bytes || color_sets < 1 || color_sets > 2) return SB_ERR_BAD_ARG;
    const int stride = color_sets > 1 ? kAccumStride2 : kAccumStride;
    *bytes = ((size_t)(P > 0 ? P : 1) * stride * sizeof(float) + kAlign - 1) / kAlign * kAlign;
    return SB_OK;
}

SB_API int sb_forward_geometry(const sb_settings* s, int P, const float* means3D, const float* opacities,
                        const float* scales, const float* rotations, const float* cov3D_precomp,
                        int32_t* radii, void* geom_ws, size_t geom_ws_bytes, int* num_rendered, void* stream) {
    if (!settings_ok(s) || P < 0 || !num_rendered) return SB_ERR_BAD_ARG;
    *num_rendered = 0;
    if (P == 0) return SB_OK;  // rasterize_points.cu:81 -- nothing launched for an empty scene
    if (!means3D || !opacities || !radii || !geom_ws) return SB_ERR_BAD_ARG;
    if (!cov3D_precomp && (!scales || !rotations)) return SB_ERR_BAD_ARG;
    size_t need = 0;
    GeometryWs g = carve_geometry(geom_ws, P, &need);
    if (geom_ws_bytes < need) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = launch_project(*s, P, means3D, opacities, scales, rotations, cov3D_precomp, radii, g, st);
    if (rc != SB_OK) return rc;
    rc = launch_depth_order(P, g, st);
    if (rc != SB_OK) return rc;
    uint32_t R = 0;
    SB_CUDA_CHECK(cudaMemcpyAsync(&R, g.offsets + (P - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    SB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (R > 0x7fffffffu) return SB_ERR_WORKSPACE;
    *num_rendered = (int)R;
    return SB_OK;
}

SB_API int sb_forward(const sb_settings* s, int P, const float* means3D, const float* opacities, const float* scales,
               const float* rotations, const float* cov3D_precomp, const float* colors, const float* colors2,
               int32_t* radii, void* geom_ws, size_t geom_ws_bytes, void* binning_ws, size_t binning_ws_bytes,
               void* image_ws, size_t image_ws_bytes, float* out_color, float* out_color2, float* out_depth,
               int* num_rendered, void* stream) {
    int rc = sb_forward_geometry(s, P, means3D, opacities, scales, rotations, cov3D_precomp, radii, geom_ws,
                                 geom_ws_bytes, num_rendered, stream);
    if (rc != SB_OK) return rc;
    size_t need = 0;
    rc = sb_binning_workspace_bytes(*num_rendered, s->image_width, s->image_height, colors2 ? 2 : 1, &need);
    if (rc != SB_OK) return rc;
    if (*num_rendered > 0 && (binning_ws == nullptr || binning_ws_bytes < need)) return SB_ERR_BINNING_TOO_SMALL;
    return sb_forward_render(s, P, *num_rendered, colors, colors2, geom_ws, geom_ws_bytes, binning_ws,
                             binning_ws_bytes, image_ws, image_ws_bytes, out_color, out_color2, out_depth, stream);
}

SB_API int sb_forward_async(const sb_settings* s, int P, const float* means3D, const float* opacities,
                     const float* scales, const float* rotations, const float* cov3D_precomp, const float* colors,
                     const float* colors2, int32_t* radii, void* geom_ws, size_t geom_ws_bytes, void* binning_ws,
                     size_t binning_ws_bytes, int capacity, void* image_ws, size_t image_ws_bytes, float* out_color,
                     float* out_color2, float* out_depth, void* stream) {
    if (!settings_ok(s) || P <= 0 || capacity < 1 || !means3D || !opacities || !radii || !geom_ws || !binning_ws ||
        !image_ws || !colors || !out_color || !out_depth)
        return SB_ERR_BAD_ARG;
    if (!cov3D_precomp && (!scales || !rotations)) return SB_ERR_BAD_ARG;
    if ((colors2 != nullptr) != (out_color2 != nullptr)) return SB_ERR_BAD_ARG;
    const int sets = colors2 ? 2 : 1;
    size_t need = 0;
    GeometryWs g = carve_geometry(geom_ws, P, &need);
    if (geom_ws_bytes < need) return SB_ERR_WORKSPACE;
    BinningWs b = carve_binning(binning_ws, capacity, tiles_of(s), sets, &need);
    if (binning_ws_bytes < need) return SB_ERR_WORKSPACE;
    ImageWs img = carve_image(image_ws, s->image_width, s->image_height, &need);
    if (image_ws_bytes < need) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = launch_project(*s, P, means3D, opacities, scales, rotations, cov3D_precomp, radii, g, st);
    if (rc != SB_OK) return rc;
    if ((rc = launch_depth_order(P, g, st)) != SB_OK) return rc;
    if ((rc = launch_finalize_count(P, g, capacity, st)) != SB_OK) return rc;
    if ((rc = launch_binning(*s, P, capacity, colors, colors2, g, b, img, g.header, st)) != SB_OK) return rc;
    return launch_blend_forward(*s, capacity, g, b, img, out_color, out_color2, out_depth, g.header + 2, st);
}

SB_API int sb_read_counts(const void* geom_ws, size_t geom_ws_bytes, int P, int* num_rendered, int* overflow,
                          void* stream) {
    if (!geom_ws || P <= 0 || !num_rendered || !overflow) return SB_ERR_BAD_ARG;
    size_t need = 0;
    GeometryWs g = carve_geometry(const_cast<void*>(geom_ws), P, &need);
    if (geom_ws_bytes < need) return SB_ERR_WORKSPACE;
    int32_t h[4] = {0, 0, 0, 0};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SB_CUDA_CHECK(cudaMemcpyAsync(h, g.header, sizeof(h), cudaMemcpyDeviceToHost, st));
    SB_CUDA_CHECK(cudaStreamSynchronize(st));
    *num_rendered = h[0];
    *overflow = h[2];
    return SB_OK;
}

SB_API int sb_forward_render(const sb_settings* s, int P, int num_rendered, const float* colors,
                      const float* colors2, const void* geom_ws, size_t geom_ws_bytes, void* binning_ws,
                      size_t binning_ws_bytes, void* image_ws, size_t image_ws_bytes, float* out_color,
                      float* out_color2, float* out_depth, void* stream) {
    if (!settings_ok(s) || P < 0 || num_rendered < 0 || !image_ws || !out_color || !out_depth) return SB_ERR_BAD_ARG;
    if (P > 0 && (!colors || !geom_ws)) return SB_ERR_BAD_ARG;
    if ((colors2 != nullptr) != (out_color2 != nullptr)) return SB_ERR_BAD_ARG;
    const int sets = colors2 ? 2 : 1;
    if (num_rendered > 0 && !binning_ws) return SB_ERR_BAD_ARG;
    size_t need = 0;
    GeometryWs g = carve_geometry(const_cast<void*>(geom_ws), P, &need);
    if (P > 0 && geom_ws_bytes < need) return SB_ERR_WORKSPACE;
    BinningWs b = carve_binning(binning_ws, num_rendered, tiles_of(s), sets, &need);
    if (num_rendered > 0 && binning_ws_bytes < need) return SB_ERR_WORKSPACE;
    ImageWs img = carve_image(image_ws, s->image_width, s->image_height, &need);
    if (image_ws_bytes < need) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = launch_binning(*s, P, num_rendered, colors, colors2, g, b, img, nullptr, st);
    if (rc != SB_OK) return rc;
    return launch_blend_forward(*s, num_rendered, g, b, img, out_color, out_color2, out_depth, nullptr, st);
}

SB_API int sb_blend_stats(const sb_settings* s, int P, int num_rendered, int sync_free, const void* geom_ws,
                          size_t geom_ws_bytes, const void* binning_ws, size_t binning_ws_bytes, const void* image_ws,
                          size_t image_ws_bytes, uint32_t* blended, uint32_t* ended, uint32_t* max_weight_bits,
                          void* stream) {
    if (!settings_ok(s) || P < 0 || num_rendered < 0) return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    if (!geom_ws || !image_ws || !blended || !ended || !max_weight_bits) return SB_ERR_BAD_ARG;
    if (num_rendered > 0 && !binning_ws) return SB_ERR_BAD_ARG;
    size_t need = 0;
    GeometryWs g = carve_geometry(const_cast<void*>(geom_ws), P, &need);
    if (geom_ws_bytes < need) return SB_ERR_WORKSPACE;
    // the one-set layout is a prefix of the two-set one, and the walk reads only that prefix
    BinningWs b = carve_binning(const_cast<void*>(binning_ws), num_rendered, tiles_of(s), 1, &need);
    if (num_rendered > 0 && binning_ws_bytes < need) return SB_ERR_WORKSPACE;
    ImageWs img = carve_image(const_cast<void*>(image_ws), s->image_width, s->image_height, &need);
    if (image_ws_bytes < need) return SB_ERR_WORKSPACE;
    if (num_rendered == 0) return SB_OK;      // every tile range is empty: nothing blended
    return launch_blend_stats(*s, b, img, sync_free ? g.header + 2 : nullptr, blended, ended, max_weight_bits,
                              static_cast<cudaStream_t>(stream));
}

SB_API int sb_backward(const sb_settings* s, int P, int num_rendered, const float* means3D, const float* colors,
                const float* scales, const float* rotations, const float* cov3D_precomp, const int32_t* radii,
                const void* geom_ws, size_t geom_ws_bytes, const void* binning_ws, size_t binning_ws_bytes,
                const void* image_ws, size_t image_ws_bytes, void* bwd_ws, size_t bwd_ws_bytes,
                const float* dL_dout_color, const float* dL_dout_color2, float* dL_dmeans3D,
                float* dL_dmeans2D, float* dL_dcolors, float* dL_dcolors2, float* dL_dopacity,
                float* dL_dscales, float* dL_drotations, float* dL_dcov3D, void* stream) {
    (void)geom_ws; (void)geom_ws_bytes;
    if ((dL_dout_color2 != nullptr) != (dL_dcolors2 != nullptr)) return SB_ERR_BAD_ARG;
    const int sets = dL_dout_color2 ? 2 : 1;
    const int stride = sets > 1 ? kAccumStride2 : kAccumStride;
    if (!settings_ok(s) || P < 0 || num_rendered < 0) return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    if (!means3D || !colors || !radii || !image_ws || !bwd_ws || !dL_dout_color || !dL_dmeans3D ||
        !dL_dmeans2D || !dL_dcolors || !dL_dopacity)
        return SB_ERR_BAD_ARG;
    if (!cov3D_precomp && (!scales || !rotations || !dL_dscales || !dL_drotations)) return SB_ERR_BAD_ARG;
    if (num_rendered > 0 && !binning_ws) return SB_ERR_BAD_ARG;
    size_t need = 0;
    BinningWs b = carve_binning(const_cast<void*>(binning_ws), num_rendered, tiles_of(s), sets, &need);
    if (num_rendered > 0 && binning_ws_bytes < need) return SB_ERR_WORKSPACE;
    ImageWs img = carve_image(const_cast<void*>(image_ws), s->image_width, s->image_height, &need);
    if (image_ws_bytes < need) return SB_ERR_WORKSPACE;
    sb_backward_workspace_bytes(P, sets, &need);
    if (bwd_ws_bytes < need) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* accum = static_cast<float*>(bwd_ws);
    { ScopedStage _p(kStAccumZero, st);
      SB_CUDA_CHECK(cudaMemsetAsync(accum, 0, (size_t)P * stride * sizeof(float), st)); }
    int rc = launch_blend_backward(*s, num_rendered, b, img, dL_dout_color, dL_dout_color2, accum, st);
    if (rc != SB_OK) return rc;
    return launch_geometry_backward(*s, P, means3D, colors, scales, rotations, cov3D_precomp, radii, accum, stride,
                                    dL_dmeans3D, dL_dmeans2D, dL_dcolors, dL_dcolors2, dL_dopacity, dL_dscales,
                                    dL_drotations, dL_dcov3D, st);
}

SB_API int sb_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    uint8_t* present, void* stream) {
    (void)projmatrix;  // the reference's test only uses the view matrix (auxiliary.h:154)
    if (P < 0) return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    if (!means3D || !viewmatrix || !present) return SB_ERR_BAD_ARG;
    return launch_mark_visible(P, means3D, viewmatrix, present, static_cast<cudaStream_t>(stream));
}

SB_API int sb_export_geometry(int P, const void* geom_ws, size_t geom_ws_bytes, float* depths, float* means2D,
                       float* conic_opacity, uint32_t* tiles_touched, void* stream) {
    if (P <= 0 || !geom_ws) return SB_ERR_BAD_ARG;
    size_t need = 0;
    GeometryWs g = carve_geometry(const_cast<void*>(geom_ws), P, &need);
    if (geom_ws_bytes < need) return SB_ERR_WORKSPACE;
    export_geometry_kernel<<<(P + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        P, g.depth_key, g.geom, g.tiles_touched, depths, means2D, conic_opacity, tiles_touched);
    SB_LAUNCH_CHECK("export_geometry_kernel");
    return SB_OK;
}

SB_API int sb_export_binning(const sb_settings* s, int P, int num_rendered, const void* geom_ws, size_t geom_ws_bytes,
                      const void* binning_ws, size_t binning_ws_bytes, const void* image_ws,
                      size_t image_ws_bytes, uint64_t* keys, uint32_t* point_list, uint32_t* ranges,
                      float* final_T, uint32_t* n_contrib, void* stream) {
    if (!settings_ok(s) || P <= 0 || num_rendered < 0 || !geom_ws || !image_ws) return SB_ERR_BAD_ARG;
    size_t need = 0;
    GeometryWs g = carve_geometry(const_cast<void*>(geom_ws), P, &need);
    if (geom_ws_bytes < need) return SB_ERR_WORKSPACE;
    const int tiles = tiles_of(s);
    BinningWs b = carve_binning(const_cast<void*>(binning_ws), num_rendered, tiles, 1, &need);
    if (num_rendered > 0 && (!binning_ws || binning_ws_bytes < need)) return SB_ERR_WORKSPACE;
    ImageWs img = carve_image(const_cast<void*>(image_ws), s->image_width, s->image_height, &need);
    if (image_ws_bytes < need) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (num_rendered > 0 && (keys || point_list)) {
        const int R = num_rendered;
        export_keys_kernel<uint32_t><<<(R + 255) / 256, 256, 0, st>>>(R, b.tile_sorted, b.point_list,
                                                                      g.depth_key, keys, point_list);
        SB_LAUNCH_CHECK("export_keys_kernel");
    }
    const size_t hw = (size_t)s->image_width * s->image_height;
    if (ranges) SB_CUDA_CHECK(cudaMemcpyAsync(ranges, img.ranges, sizeof(uint2) * (size_t)tiles, cudaMemcpyDeviceToDevice, st));
    if (final_T) SB_CUDA_CHECK(cudaMemcpyAsync(final_T, img.final_T, sizeof(float) * hw, cudaMemcpyDeviceToDevice, st));
    if (n_contrib) SB_CUDA_CHECK(cudaMemcpyAsync(n_contrib, img.n_contrib, sizeof(uint32_t) * hw, cudaMemcpyDeviceToDevice, st));
    return SB_OK;
}

SB_API int sb_export_cover(const sb_settings* s, int num_rendered, const void* binning_ws, size_t binning_ws_bytes,
                           uint8_t* cover, void* stream) {
    if (!settings_ok(s) || num_rendered < 0 || (num_rendered > 0 && !cover)) return SB_ERR_BAD_ARG;
    if (num_rendered == 0) return SB_OK;
    size_t need = 0;
    BinningWs b = carve_binning(const_cast<void*>(binning_ws), num_rendered, tiles_of(s), 1, &need);
    if (!binning_ws || binning_ws_bytes < need) return SB_ERR_WORKSPACE;
    export_cover_kernel<<<(num_rendered + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(num_rendered,
                                                                                                  b.recA, cover);
    SB_LAUNCH_CHECK("export_cover_kernel");
    return SB_OK;
}

SB_API int sb_radix_sort_temp_bytes(int capacity, int bits, size_t* bytes) {
    if (!bytes || capacity < 0 || capacity >= (1 << 30) || bits < 1 || bits > 32) return SB_ERR_BAD_ARG;
    *bytes = radix_temp_bytes(capacity, bits);
    return SB_OK;
}

SB_API int sb_radix_sort_pairs(const uint32_t* keys_in, const uint32_t* vals_in, uint32_t* keys_out, uint32_t* vals_out,
                               int capacity, const int32_t* n_dev, int begin_bit, int end_bit, void* temp,
                               size_t temp_bytes, void* stream) {
    if (capacity < 0 || capacity >= (1 << 30) || begin_bit < 0 || end_bit > 32 || begin_bit >= end_bit)
        return SB_ERR_BAD_ARG;
    if (capacity == 0) return SB_OK;
    if (!keys_in || !keys_out || !vals_out || !temp) return SB_ERR_BAD_ARG;
    // a pass may write an output while it reads the inputs, so no output may be an input or the other output
    if (keys_out == keys_in || vals_out == keys_in || keys_out == vals_out ||
        (vals_in && (keys_out == vals_in || vals_out == vals_in)))
        return SB_ERR_BAD_ARG;
    return radix_sort_pairs(keys_in, vals_in, keys_out, vals_out, capacity, n_dev, begin_bit, end_bit, temp, temp_bytes,
                            static_cast<cudaStream_t>(stream));
}

SB_API int sb_profile_begin(void) {
    for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    g_prof.clear();
    g_prof_on = true;
    return SB_OK;
}

SB_API int sb_profile_end(float* stage_ms, int* stage_calls) {
    g_prof_on = false;
    if (!stage_ms || !stage_calls) return SB_ERR_BAD_ARG;
    for (int i = 0; i < kNumStages; ++i) { stage_ms[i] = 0.f; stage_calls[i] = 0; }
    SB_CUDA_CHECK(cudaDeviceSynchronize());
    for (auto& r : g_prof) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { stage_ms[r.stage] += ms; stage_calls[r.stage]++; }
        cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    }
    g_prof.clear();
    return SB_OK;
}

SB_API const char* sb_stage_name(int stage) {
    static const char* names[kNumStages] = {"project", "depth_sort", "depth_scan", "emit_instances", "tile_sort",
                                            "ranges_records", "blend_forward", "accum_zero", "blend_backward",
                                            "geometry_backward"};
    return (stage >= 0 && stage < kNumStages) ? names[stage] : "?";
}

}  // extern "C"
