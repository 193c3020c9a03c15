// Frame resize on the device: uint8 [n, in_h, in_w, 3] -> the crop window of the resized frames,
// uint8 [n, crop_h, crop_w, 3] (vcl_resize_frames).
//
// VCL_RESIZE_NEAREST: torch.nn.functional.interpolate(mode="nearest") on CPU tensors, which
//   load_video (video_chatgpt/eval/model_utils.py:39-44) runs on the float copy of its frames; the values are
//   integers there, so a uint8 gather is exact:  s = fp32(in) / fp32(out), src = min(floor(fp32(dst) * s), in - 1).
// VCL_RESIZE_BICUBIC: PIL.Image.resize(..., BICUBIC) on RGB frames, the resize of CLIPImageProcessor
//   (libImaging/Resample.c): a horizontal pass, then a vertical one, each rounding to uint8 and skipped when its
//   size does not change. Output index xx of a pass takes the source span [xmin, xmin + n) with int32 weights
//   (22 fraction bits) computed in double arithmetic (resize_window / resize_coeffs_kernel); a pixel is
//   clamp((2^21 + sum(p k)) >> 22, 0, 255).
//
// Only the crop window is computed: the horizontal pass produces the crop columns of the source rows the crop
// rows' vertical spans touch (rows r0 .. r0 + rows - 1), the vertical pass the crop rows from them. The weight
// tables and that intermediate live in the caller's workspace (resize_frames_workspace gives its size); the
// tables are built on the device, so a call neither synchronises nor allocates.
//
// Bandwidth-bound and small next to the tower: a thread owns one output pixel and reads its taps through L1/L2
// (neighbouring threads share all but one or two source pixels).
#include <math.h>

#include "../../include/vcl.h"
#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

constexpr int RESIZE_MAX = 8192;        // largest accepted frame count, frame side and output side
constexpr int PRECISION_BITS = 22;      // PIL's fixed point for 8-bit images: 32 - 8 - 2
constexpr int RESIZE_THREADS = 128;

// PIL's double arithmetic, operation by operation: the intrinsics keep nvcc from contracting a multiply and an
// add into an FMA, which would round once instead of twice. The host side (the workspace size) uses the same
// functions, compiled for x86-64 without FMA.
__host__ __device__ __forceinline__ double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double ddiv(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

struct Span {
  double scale, fs, support, center;   // fs = max(scale, 1): the filter's stretch
  int xmin, n;
};

// The source span of output index xx when n_in samples become n_out (PIL's precompute_coeffs).
__host__ __device__ __forceinline__ Span resize_window(int n_in, int n_out, int xx) {
  Span s;
  s.scale = ddiv((double)n_in, (double)n_out);
  s.fs = s.scale < 1.0 ? 1.0 : s.scale;
  s.support = dmul(2.0, s.fs);
  s.center = dmul(dadd((double)xx, 0.5), s.scale);
  s.xmin = (int)dadd(dadd(s.center, -s.support), 0.5);
  if (s.xmin < 0) s.xmin = 0;
  int xmax = (int)dadd(dadd(s.center, s.support), 0.5);
  if (xmax > n_in) xmax = n_in;
  s.n = xmax - s.xmin;
  return s;
}

// Taps per table row: PIL's ksize = 2 * ceil(support) + 1, an upper bound of every span's n.
int resize_taps(int n_in, int n_out) {
  const double scale = (double)n_in / (double)n_out;
  return (int)ceil(2.0 * (scale < 1.0 ? 1.0 : scale)) * 2 + 1;
}

__device__ __forceinline__ double bicubic_filter(double x) {   // a = -0.5
  if (x < 0.0) x = -x;
  if (x < 1.0) return dadd(dmul(dmul(dadd(dmul(1.5, x), -2.5), x), x), 1.0);
  if (x < 2.0) return dmul(dadd(dmul(dadd(dmul(dadd(x, -5.0), x), 8.0), x), -4.0), -0.5);
  return 0.0;
}

struct Table {
  int n_in, n_out, first, count, taps;   // output indices first .. first + count - 1
  int2* bounds;                          // [count] (xmin, n)
  int* k;                                // [count][taps]
};

// Thread i builds row i of the horizontal table, then of the vertical one (bounds + fixed-point weights).
__global__ void __launch_bounds__(RESIZE_THREADS) resize_coeffs_kernel(Table th, Table tv) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  Table t = th;
  if (i >= th.count) { i -= th.count; t = tv; }
  if (i >= t.count) return;
  const int xx = t.first + i;
  const Span s = resize_window(t.n_in, t.n_out, xx);
  const double ss = ddiv(1.0, s.fs);
  const int n = min(s.n, t.taps);
  // weight of tap x: cubic((x + xmin - center + 0.5) * ss); the sum runs in tap order like PIL's
  double ww = 0.0;
  for (int x = 0; x < n; ++x) ww = dadd(ww, bicubic_filter(dmul(dadd(dadd((double)(x + s.xmin), -s.center), 0.5), ss)));
  int* k = t.k + (long long)i * t.taps;
  for (int x = 0; x < t.taps; ++x) {
    int q = 0;
    if (x < n) {
      double w = bicubic_filter(dmul(dadd(dadd((double)(x + s.xmin), -s.center), 0.5), ss));
      if (ww != 0.0) w = ddiv(w, ww);
      const double f = dmul(w, (double)(1 << PRECISION_BITS));       // exact: a power of two
      q = (int)(w < 0 ? dadd(-0.5, f) : dadd(0.5, f));                 // truncation: half away from zero
    }
    k[x] = q;
  }
  t.bounds[i] = make_int2(s.xmin, n);
}

__device__ __forceinline__ uint8_t clip8(int acc) {
  acc >>= PRECISION_BITS;
  return (uint8_t)(acc < 0 ? 0 : acc > 255 ? 255 : acc);
}

// dst row y, column x of frame z = the horizontal filter of table row x over src row y.
__global__ void __launch_bounds__(RESIZE_THREADS)
resize_h_kernel(const uint8_t* __restrict__ src, long long src_frame, int src_row, uint8_t* __restrict__ dst,
                long long dst_frame, int dst_row, int cols, const int2* __restrict__ bounds,
                const int* __restrict__ kk, int taps) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= cols) return;
  const uint8_t* s = src + blockIdx.z * src_frame + (long long)blockIdx.y * src_row;
  const int2 b = bounds[x];
  const int* k = kk + (long long)x * taps;
  int a0 = 1 << (PRECISION_BITS - 1), a1 = a0, a2 = a0;
  s += 3 * b.x;
  for (int t = 0; t < b.y; ++t, s += 3) {
    const int w = k[t];
    a0 += s[0] * w;
    a1 += s[1] * w;
    a2 += s[2] * w;
  }
  uint8_t* d = dst + blockIdx.z * dst_frame + (long long)blockIdx.y * dst_row + 3 * x;
  d[0] = clip8(a0);
  d[1] = clip8(a1);
  d[2] = clip8(a2);
}

// dst row y, column x of frame z = the vertical filter of table row y over column x of src rows
// (ymin - r0) .. (ymin - r0 + n - 1); src holds `rows` rows.
__global__ void __launch_bounds__(RESIZE_THREADS)
resize_v_kernel(const uint8_t* __restrict__ src, long long src_frame, int src_row, int r0, int rows,
                uint8_t* __restrict__ dst, long long dst_frame, int dst_row, int cols, const int2* __restrict__ bounds,
                const int* __restrict__ kk, int taps) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= cols) return;
  const int y = blockIdx.y;
  const int2 b = bounds[y];
  const int* k = kk + (long long)y * taps;
  const uint8_t* s = src + blockIdx.z * src_frame + 3 * x;
  int a0 = 1 << (PRECISION_BITS - 1), a1 = a0, a2 = a0;
  for (int t = 0; t < b.y; ++t) {
    const int r = b.x - r0 + t;
    if (r < 0 || r >= rows) continue;   // never taken: the workspace was sized from the same spans
    const uint8_t* p = s + (long long)r * src_row;
    const int w = k[t];
    a0 += p[0] * w;
    a1 += p[1] * w;
    a2 += p[2] * w;
  }
  uint8_t* d = dst + blockIdx.z * dst_frame + (long long)y * dst_row + 3 * x;
  d[0] = clip8(a0);
  d[1] = clip8(a1);
  d[2] = clip8(a2);
}

// torch's nearest index rule (aten/src/ATen/native/UpSample.h: nearest_idx with the scale in/out); with
// out == in it is the identity, which makes this kernel the crop copy as well.
__device__ __forceinline__ int nearest_src(int dst, float s, int n_in) {
  return min((int)floorf(__fmul_rn((float)dst, s)), n_in - 1);
}

__global__ void __launch_bounds__(RESIZE_THREADS)
resize_nearest_kernel(const uint8_t* __restrict__ src, long long src_frame, int in_h, int in_w, float sh, float sw,
                      int top, int left, uint8_t* __restrict__ dst, long long dst_frame, int cols) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= cols) return;
  const int y = blockIdx.y;
  const int sy = nearest_src(top + y, sh, in_h), sx = nearest_src(left + x, sw, in_w);
  const uint8_t* p = src + blockIdx.z * src_frame + ((long long)sy * in_w + sx) * 3;
  uint8_t* d = dst + blockIdx.z * dst_frame + ((long long)y * cols + x) * 3;
  d[0] = p[0];
  d[1] = p[1];
  d[2] = p[2];
}

constexpr size_t WS_ALIGN = 256;
inline size_t align_up(size_t b) { return (b + WS_ALIGN - 1) / WS_ALIGN * WS_ALIGN; }

// The geometry of one call, checked, and where each piece of the workspace goes.
struct Plan {
  bool h_pass = false, v_pass = false;
  int taps_h = 0, taps_v = 0;
  int r0 = 0, rows = 0;                 // source rows the horizontal pass produces (vertical pass needed)
  size_t off_bh = 0, off_kh = 0, off_bv = 0, off_kv = 0, off_mid = 0, bytes = 0;
};

int plan_resize(int n, int in_h, int in_w, int mode, int out_h, int out_w, int crop_top, int crop_left, int crop_h,
                int crop_w, Plan* p) {
  VCL_REQUIRE(mode == VCL_RESIZE_NEAREST || mode == VCL_RESIZE_BICUBIC,
              "vcl_resize_frames: unknown mode %d (VCL_RESIZE_NEAREST=0, VCL_RESIZE_BICUBIC=1)", mode);
  VCL_REQUIRE(n >= 1 && n <= RESIZE_MAX, "vcl_resize_frames: n=%d frames (1..%d)", n, RESIZE_MAX);
  VCL_REQUIRE(in_h >= 1 && in_h <= RESIZE_MAX && in_w >= 1 && in_w <= RESIZE_MAX,
              "vcl_resize_frames: in_h x in_w = %d x %d (each 1..%d)", in_h, in_w, RESIZE_MAX);
  VCL_REQUIRE(out_h >= 1 && out_h <= RESIZE_MAX && out_w >= 1 && out_w <= RESIZE_MAX,
              "vcl_resize_frames: out_h x out_w = %d x %d (each 1..%d)", out_h, out_w, RESIZE_MAX);
  VCL_REQUIRE(crop_h >= 1 && crop_w >= 1, "vcl_resize_frames: crop_h x crop_w = %d x %d (each >= 1)", crop_h, crop_w);
  VCL_REQUIRE(crop_top >= 0 && crop_top <= out_h - crop_h && crop_left >= 0 && crop_left <= out_w - crop_w,
              "vcl_resize_frames: crop (crop_top=%d, crop_left=%d, crop_h=%d, crop_w=%d) lies outside the %d x %d "
              "resized frame", crop_top, crop_left, crop_h, crop_w, out_h, out_w);
  *p = Plan();
  if (mode == VCL_RESIZE_NEAREST) return 0;
  p->h_pass = out_w != in_w;
  p->v_pass = out_h != in_h;
  size_t b = 0;
  if (p->h_pass) {
    p->taps_h = resize_taps(in_w, out_w);
    p->off_bh = b; b = align_up(b + (size_t)crop_w * sizeof(int2));
    p->off_kh = b; b = align_up(b + (size_t)crop_w * p->taps_h * sizeof(int));
  }
  if (p->v_pass) {
    p->taps_v = resize_taps(in_h, out_h);
    p->off_bv = b; b = align_up(b + (size_t)crop_h * sizeof(int2));
    p->off_kv = b; b = align_up(b + (size_t)crop_h * p->taps_v * sizeof(int));
    // the spans only move forward with the output index: the first and last crop rows bound them all
    const Span first = resize_window(in_h, out_h, crop_top), last = resize_window(in_h, out_h, crop_top + crop_h - 1);
    p->r0 = first.xmin;
    p->rows = last.xmin + last.n - first.xmin;
    if (p->h_pass) { p->off_mid = b; b = align_up(b + (size_t)n * p->rows * crop_w * 3); }
  }
  p->bytes = b;
  return 0;
}

inline dim3 grid_of(int cols, int rows, int n) { return dim3((cols + RESIZE_THREADS - 1) / RESIZE_THREADS, rows, n); }

}  // namespace

size_t resize_frames_workspace(int n, int in_h, int in_w, int mode, int out_h, int out_w, int crop_top, int crop_left,
                               int crop_h, int crop_w) {
  Plan p;
  if (plan_resize(n, in_h, in_w, mode, out_h, out_w, crop_top, crop_left, crop_h, crop_w, &p) != 0) return SIZE_MAX;
  return p.bytes;
}

int launch_resize_frames(const uint8_t* in, int n, int in_h, int in_w, int mode, int out_h, int out_w, int crop_top,
                         int crop_left, int crop_h, int crop_w, uint8_t* out, void* ws, size_t ws_bytes,
                         cudaStream_t stream) {
  Plan p;
  if (plan_resize(n, in_h, in_w, mode, out_h, out_w, crop_top, crop_left, crop_h, crop_w, &p) != 0) return -1;
  VCL_REQUIRE(ws_bytes >= p.bytes, "vcl_resize_frames: ws_bytes=%zu but this resize needs %zu "
              "(vcl_resize_frames_workspace_bytes)", ws_bytes, p.bytes);
  VCL_REQUIRE(p.bytes == 0 || ws, "vcl_resize_frames: null ws (this resize needs %zu bytes)", p.bytes);
  VCL_REQUIRE(p.bytes == 0 || (uintptr_t)ws % 16 == 0, "vcl_resize_frames: ws must be 16-byte aligned");
  const long long in_frame = (long long)in_h * in_w * 3, out_frame = (long long)crop_h * crop_w * 3;
  const int in_row = in_w * 3, out_row = crop_w * 3;

  if (!p.h_pass && !p.v_pass) {   // nearest, or a bicubic resize to the same size: PIL copies, the crop remains
    const float sh = (float)in_h / (float)out_h, sw = (float)in_w / (float)out_w;   // IEEE fp32, as torch
    resize_nearest_kernel<<<grid_of(crop_w, crop_h, n), RESIZE_THREADS, 0, stream>>>(
        in, in_frame, in_h, in_w, sh, sw, crop_top, crop_left, out, out_frame, crop_w);
    VCL_CUDA_OK(cudaGetLastError());
    count_launches(1);
    return 0;
  }

  uint8_t* w = static_cast<uint8_t*>(ws);
  Table th{in_w, out_w, crop_left, p.h_pass ? crop_w : 0, p.taps_h, reinterpret_cast<int2*>(w + p.off_bh),
           reinterpret_cast<int*>(w + p.off_kh)};
  Table tv{in_h, out_h, crop_top, p.v_pass ? crop_h : 0, p.taps_v, reinterpret_cast<int2*>(w + p.off_bv),
           reinterpret_cast<int*>(w + p.off_kv)};
  resize_coeffs_kernel<<<(th.count + tv.count + RESIZE_THREADS - 1) / RESIZE_THREADS, RESIZE_THREADS, 0, stream>>>(th, tv);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);

  if (p.h_pass) {
    // without a vertical pass the horizontal one writes the crop rows straight into out
    const bool direct = !p.v_pass;
    const uint8_t* src = in + (long long)(direct ? crop_top : p.r0) * in_row;
    uint8_t* dst = direct ? out : w + p.off_mid;
    const int rows = direct ? crop_h : p.rows;
    const long long dst_frame = direct ? out_frame : (long long)p.rows * out_row;
    resize_h_kernel<<<grid_of(crop_w, rows, n), RESIZE_THREADS, 0, stream>>>(src, in_frame, in_row, dst, dst_frame,
                                                                            out_row, crop_w, th.bounds, th.k, th.taps);
    VCL_CUDA_OK(cudaGetLastError());
    count_launches(1);
  }
  if (p.v_pass) {
    // the vertical pass reads the intermediate, or the input's crop columns when the width is unchanged
    const uint8_t* src = p.h_pass ? w + p.off_mid : in + (long long)p.r0 * in_row + 3 * crop_left;
    const long long src_frame = p.h_pass ? (long long)p.rows * out_row : in_frame;
    const int src_row = p.h_pass ? out_row : in_row;
    resize_v_kernel<<<grid_of(crop_w, crop_h, n), RESIZE_THREADS, 0, stream>>>(
        src, src_frame, src_row, p.r0, p.rows, out, out_frame, out_row, crop_w, tv.bounds, tv.k, tv.taps);
    VCL_CUDA_OK(cudaGetLastError());
    count_launches(1);
  }
  return 0;
}

}  // namespace vcl
