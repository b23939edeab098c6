// ingest.cu -- one RGB-D frame as the dataset readers decode it (uint8 RGB HWC, uint16 depth) turned into the
// model-ready tensors, in one launch: colour [3,H,W] float32 in [0,1] and depth [1,H,W] float32 in metres.
// It restates the reference loader's per-frame host work (R/datasets/gradslam_datasets/basedataset.py:224-257,
// 296-341, then splatam.py's permute(2,0,1) / 255):
//   colour = float32(cv2.resize(float64 rgb, INTER_LINEAR)) / 255
//   depth  = float32(cv2.resize(float64 raw, INTER_NEAREST) / png_depth_scale)
// with cv2's rules (oracle/ingest_numpy.py restates them in numpy): an equal size is a copy; an exact 2x downscale in
// both axes is cv2's INTER_AREA (2x2 box mean), which cv2 substitutes for INTER_LINEAR there; otherwise bilinear with
// half-pixel centres, evaluated in double, horizontal pass first, edge taps clamped with weight 0.  Every double
// operation is an explicit _rn intrinsic so that no multiply-add is contracted into an FMA: the result is then the
// same double the numpy restatement computes, and its float32 rounding is the same bit pattern.
// Per output pixel the kernel reads 3 B of colour and 2 B of depth (12 B of colour at an exact 2x downscale, up to
// 12 B through the bilinear footprint, mostly from L1/L2) and writes 16 B.
// The second half holds the live-capture kernels (capture.py): the online demo converts a phone packet with cv2 on
// uint8 colour and float32 depth, whose fixed-point rules differ from the float64 ones above.
#include "common.cuh"

namespace sb {

namespace {

constexpr int kIngestBX = 32, kIngestBY = 8;

struct Axis {            // one bilinear axis: source taps i0/i1 and weights w0/w1
    int i0, i1;
    double w0, w1;
};

__device__ __forceinline__ Axis linear_axis(int d, int n_src, double scale) {
    double f = __dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5);
    const double fl = floor(f);
    const int i = (int)fl;
    f = __dsub_rn(f, fl);
    Axis a;
    if (i < 0 || i >= n_src - 1) {
        a.i0 = a.i1 = i < 0 ? 0 : n_src - 1;
        a.w0 = 1.0; a.w1 = 0.0;
    } else {
        a.i0 = i; a.i1 = i + 1;
        a.w0 = __dsub_rn(1.0, f); a.w1 = f;
    }
    return a;
}

__device__ __forceinline__ double lerp2(double v0, double w0, double v1, double w1) {
    return __dadd_rn(__dmul_rn(v0, w0), __dmul_rn(v1, w1));
}

// mode 0: copy, 1: exact 2x box, 2: bilinear
__global__ void __launch_bounds__(kIngestBX * kIngestBY)
ingest_rgbd_kernel(const uint8_t* __restrict__ rgb, int hc, int wc, const uint16_t* __restrict__ depth, int hd,
                   int wd, int H, int W, int mode, double scale_x, double scale_y, double near_x, double near_y,
                   double png_depth_scale, float* __restrict__ color_out, float* __restrict__ depth_out) {
    const int x = blockIdx.x * kIngestBX + threadIdx.x;
    const int y = blockIdx.y * kIngestBY + threadIdx.y;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, o = (size_t)y * W + x;

    double c[3];
    if (mode == 0) {
        const uint8_t* p = rgb + ((size_t)y * wc + x) * 3;
        for (int k = 0; k < 3; ++k) c[k] = (double)p[k];
    } else if (mode == 1) {
        const uint8_t* r0 = rgb + ((size_t)(2 * y) * wc + 2 * x) * 3;
        const uint8_t* r1 = r0 + (size_t)wc * 3;
        for (int k = 0; k < 3; ++k)      // integer sums of at most 4 * 255: exact in any order
            c[k] = __dmul_rn((double)((int)r0[k] + r0[k + 3] + r1[k] + r1[k + 3]), 0.25);
    } else {
        const Axis ax = linear_axis(x, wc, scale_x), ay = linear_axis(y, hc, scale_y);
        const uint8_t* r0 = rgb + (size_t)ay.i0 * wc * 3;
        const uint8_t* r1 = rgb + (size_t)ay.i1 * wc * 3;
        for (int k = 0; k < 3; ++k) {
            const double h0 = lerp2((double)r0[ax.i0 * 3 + k], ax.w0, (double)r0[ax.i1 * 3 + k], ax.w1);
            const double h1 = lerp2((double)r1[ax.i0 * 3 + k], ax.w0, (double)r1[ax.i1 * 3 + k], ax.w1);
            c[k] = lerp2(h0, ay.w0, h1, ay.w1);
        }
    }
    for (int k = 0; k < 3; ++k) color_out[k * HW + o] = __fdiv_rn(__double2float_rn(c[k]), 255.0f);

    int sx = (int)floor(__dmul_rn((double)x, near_x)), sy = (int)floor(__dmul_rn((double)y, near_y));
    sx = sx < wd - 1 ? sx : wd - 1;
    sy = sy < hd - 1 ? sy : hd - 1;
    depth_out[o] = __double2float_rn(__ddiv_rn((double)depth[(size_t)sy * wd + sx], png_depth_scale));
}

// ---- live capture packets (R/scripts/iphone_demo.py:218-243, nerfcapture2dataset.py:133-138) ------------------------
// Colour is cv2.resize on uint8, which runs in fixed point (oracle/capture_numpy.py: resize_linear_u8): per axis the
// source coordinate is rounded to float32, the two weights to integers of 2^11, the horizontal pass sums in int32 and
// the vertical pass uses the vectorised rounding of cv2's VResizeLinearVec_32s8u.

struct AxisQ {           // one fixed-point bilinear axis: taps i0/i1 and weights w0/w1 in units of 2^-11
    int i0, i1, w0, w1;
};

// horizontal: an edge tap is clamped with weight 0 on the second tap; vertical: both taps are clamped and the weights
// kept (cv2 clamps the row index only), which differs at the clamped rows of an upscale
__device__ __forceinline__ AxisQ linear_axis_q(int d, int n_src, double scale, bool horizontal) {
    float fx = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
    const float fl = floorf(fx);
    const int sx = (int)fl;
    fx = __fsub_rn(fx, fl);
    AxisQ a;
    if (!horizontal) {
        a.i0 = min(max(sx, 0), n_src - 1);
        a.i1 = min(max(sx + 1, 0), n_src - 1);
    } else if (sx < 0 || sx >= n_src - 1) {
        a.i0 = a.i1 = sx < 0 ? 0 : n_src - 1;
        fx = 0.f;
    } else {
        a.i0 = sx; a.i1 = sx + 1;
    }
    a.w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f));
    a.w1 = __float2int_rn(__fmul_rn(fx, 2048.f));
    return a;
}

__device__ __forceinline__ int nearest_tap(int d, double scale, int n_src) {
    const int s = (int)floor(__dmul_rn((double)d, scale));
    return s < n_src - 1 ? s : n_src - 1;
}

// mode 0: copy, 1: exact 2x box (cv2's INTER_AREA substitution), 2: fixed-point bilinear
__global__ void __launch_bounds__(kIngestBX * kIngestBY)
ingest_capture_kernel(const uint8_t* __restrict__ rgb, int hc, int wc, const float* __restrict__ depth, int hd, int wd,
                      int H, int W, int mode, double scale_x, double scale_y, double near_x, double near_y,
                      float* __restrict__ color_out, float* __restrict__ depth_out) {
    const int x = blockIdx.x * kIngestBX + threadIdx.x;
    const int y = blockIdx.y * kIngestBY + threadIdx.y;
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W, o = (size_t)y * W + x;

    int c[3];
    if (mode == 0) {
        const uint8_t* p = rgb + ((size_t)y * wc + x) * 3;
        for (int k = 0; k < 3; ++k) c[k] = p[k];
    } else if (mode == 1) {
        const uint8_t* r0 = rgb + ((size_t)(2 * y) * wc + 2 * x) * 3;
        const uint8_t* r1 = r0 + (size_t)wc * 3;
        for (int k = 0; k < 3; ++k) c[k] = ((int)r0[k] + r0[k + 3] + r1[k] + r1[k + 3] + 2) >> 2;
    } else {
        const AxisQ ax = linear_axis_q(x, wc, scale_x, true), ay = linear_axis_q(y, hc, scale_y, false);
        const uint8_t* r0 = rgb + (size_t)ay.i0 * wc * 3;
        const uint8_t* r1 = rgb + (size_t)ay.i1 * wc * 3;
        for (int k = 0; k < 3; ++k) {
            const int h0 = r0[ax.i0 * 3 + k] * ax.w0 + r0[ax.i1 * 3 + k] * ax.w1;
            const int h1 = r1[ax.i0 * 3 + k] * ax.w0 + r1[ax.i1 * 3 + k] * ax.w1;
            const int v = ((((h0 >> 4) * ay.w0) >> 16) + (((h1 >> 4) * ay.w1) >> 16) + 2) >> 2;
            c[k] = v < 0 ? 0 : (v > 255 ? 255 : v);
        }
    }
    for (int k = 0; k < 3; ++k) color_out[k * HW + o] = __fdiv_rn((float)c[k], 255.0f);

    // float32 passes through bit for bit (NaN and negative values included)
    depth_out[o] = depth[(size_t)nearest_tap(y, near_y, hd) * wd + nearest_tap(x, near_x, wd)];
}

// numpy's float32 -> uint16 cast on x86-64: a truncating conversion to int32 (cvttss2si), whose out-of-range and NaN
// result is INT_MIN, then the low 16 bits
__device__ __forceinline__ uint16_t quantise_u16(float d, float depth_scale) {
    const float v = __fdiv_rn(__fmul_rn(d, 65535.0f), depth_scale);
    const int i = (v > -2147483648.0f && v < 2147483648.0f) ? __float2int_rz(v) : INT_MIN;
    return (uint16_t)(i & 0xffff);
}

__global__ void __launch_bounds__(kIngestBX * kIngestBY)
capture_depth_u16_kernel(const float* __restrict__ depth, int hd, int wd, float depth_scale, int H, int W,
                         double near_x, double near_y, uint16_t* __restrict__ out) {
    const int x = blockIdx.x * kIngestBX + threadIdx.x;
    const int y = blockIdx.y * kIngestBY + threadIdx.y;
    if (x >= W || y >= H) return;
    out[(size_t)y * W + x] =
        quantise_u16(depth[(size_t)nearest_tap(y, near_y, hd) * wd + nearest_tap(x, near_x, wd)], depth_scale);
}

bool capture_sizes_ok(int hd, int wd, int H, int W) {
    return hd >= 1 && wd >= 1 && H >= 1 && W >= 1 && H <= 65535 * kIngestBY &&
           (long long)H * W <= (long long)INT_MAX && (long long)hd * wd <= (long long)INT_MAX;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_ingest_rgbd(const uint8_t* rgb, int color_height, int color_width, const uint16_t* depth,
                          int depth_height, int depth_width, int height, int width, double png_depth_scale,
                          float* color_out, float* depth_out, void* stream) {
    if (!rgb || !depth || !color_out || !depth_out || color_height < 1 || color_width < 1 || depth_height < 1 ||
        depth_width < 1 || height < 1 || width < 1 || !(png_depth_scale > 0.0) ||
        height > 65535 * kIngestBY)
        return SB_ERR_BAD_ARG;
    const int mode = (color_height == height && color_width == width) ? 0
                   : (color_height == 2 * height && color_width == 2 * width) ? 1 : 2;
    // cv2: inv_scale = dst / src, scale = 1 / inv_scale, both in double
    const double scale_x = 1.0 / ((double)width / color_width), scale_y = 1.0 / ((double)height / color_height);
    const double near_x = 1.0 / ((double)width / depth_width), near_y = 1.0 / ((double)height / depth_height);
    const dim3 block(kIngestBX, kIngestBY), grid((width + kIngestBX - 1) / kIngestBX, (height + kIngestBY - 1) / kIngestBY);
    ingest_rgbd_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
        rgb, color_height, color_width, depth, depth_height, depth_width, height, width, mode, scale_x, scale_y, near_x,
        near_y, png_depth_scale, color_out, depth_out);
    SB_LAUNCH_CHECK("ingest_rgbd_kernel");
    return SB_OK;
}

SB_API int sb_ingest_capture(const uint8_t* rgb, int color_height, int color_width, const float* depth,
                             int depth_height, int depth_width, int height, int width, float* color_out,
                             float* depth_out, void* stream) {
    if (!rgb || !depth || !color_out || !depth_out || color_height < 1 || color_width < 1 ||
        !capture_sizes_ok(depth_height, depth_width, height, width) ||
        (long long)color_height * color_width * 3 > (long long)INT_MAX)
        return SB_ERR_BAD_ARG;
    const int mode = (color_height == height && color_width == width) ? 0
                   : (color_height == 2 * height && color_width == 2 * width) ? 1 : 2;
    const double scale_x = 1.0 / ((double)width / color_width), scale_y = 1.0 / ((double)height / color_height);
    const double near_x = 1.0 / ((double)width / depth_width), near_y = 1.0 / ((double)height / depth_height);
    const dim3 block(kIngestBX, kIngestBY), grid((width + kIngestBX - 1) / kIngestBX, (height + kIngestBY - 1) / kIngestBY);
    ingest_capture_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
        rgb, color_height, color_width, depth, depth_height, depth_width, height, width, mode, scale_x, scale_y, near_x,
        near_y, color_out, depth_out);
    SB_LAUNCH_CHECK("ingest_capture_kernel");
    return SB_OK;
}

SB_API int sb_capture_depth_u16(const float* depth, int depth_height, int depth_width, float depth_scale, int height,
                                int width, uint16_t* out, void* stream) {
    if (!depth || !out || !capture_sizes_ok(depth_height, depth_width, height, width) || !(depth_scale > 0.f) ||
        !(depth_scale < INFINITY))
        return SB_ERR_BAD_ARG;
    const double near_x = 1.0 / ((double)width / depth_width), near_y = 1.0 / ((double)height / depth_height);
    const dim3 block(kIngestBX, kIngestBY), grid((width + kIngestBX - 1) / kIngestBX, (height + kIngestBY - 1) / kIngestBY);
    capture_depth_u16_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
        depth, depth_height, depth_width, depth_scale, height, width, near_x, near_y, out);
    SB_LAUNCH_CHECK("capture_depth_u16_kernel");
    return SB_OK;
}

}  // extern "C"
