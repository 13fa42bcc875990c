// Depth bilateral pre-filter (SURVEY.md §8(f)2).  BundleFusion filters every depth map before integration
// (Server/tools/recons/zParametersBundlingScanNet.txt:72-74: sigmaD 2.0 px, sigmaR 0.05 m, enabled); the only in-tree
// statement of that kernel is bilateralFilterFloatMapDevice in
// /root/reference/AnnotationTools/Filter2dAnnotations/filter.cu:210-247 (with gaussD/gaussR at :191-208), one thread per
// pixel on global memory.  Arithmetic reproduced as written there: radius = ceil(2*sigmaD); domain weight
// expf(-((dx*dx+dy*dy) / (2.0f*sigmaD*sigmaD))) in float; range weight exp(-(dd*dd) / (2.0*sigmaR*sigmaR)) in DOUBLE,
// rounded to float; taps visited x-outer / y-inner; sum += w*depth contracted to an FMA (the reference's nvcc default);
// MINF (-inf) marks invalid input and output.  exp/expf are not correctly rounded and differ between CUDA releases and
// from libm, so parity with the CPU restatement is to a stated tolerance (tests/test_filter_gpu.py), not bit-exact.
// Layout here: the (2r+1)^2 domain weights are computed once per CTA into shared memory and the 16x16 tile plus its
// halo is staged in shared memory (the reference re-reads global memory 81 times per pixel).
#include "tsdf_internal.cuh"

using namespace scn_tsdf_detail;

namespace {

constexpr int kTile = 16;
constexpr int kMaxRadius = 8;

__global__ void k_depth_to_metres_minf(const uint16_t* __restrict__ src, const BatchParams bp, float depth_shift, size_t frame_px, float* __restrict__ out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const int k = blockIdx.y;
  if (i >= frame_px) return;
  const uint16_t raw = src[(size_t)bp.f[k].src * frame_px + i];
  out[(size_t)k * frame_px + i] = raw == 0 ? -INFINITY : __fdiv_rn((float)raw, depth_shift);   // Filter2dAnnotations.cpp:245-256
}

__global__ void __launch_bounds__(kTile * kTile)
k_bilateral(const float* __restrict__ in, float* __restrict__ out, int W, int H, float sigmaD, float sigmaR, int radius) {
  __shared__ float s_tile[(kTile + 2 * kMaxRadius) * (kTile + 2 * kMaxRadius)];
  __shared__ float s_gd[(2 * kMaxRadius + 1) * (2 * kMaxRadius + 1)];
  const size_t frame = (size_t)blockIdx.z * W * H;
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTile + tx;
  const int x0 = blockIdx.x * kTile - radius, y0 = blockIdx.y * kTile - radius;
  const int span = kTile + 2 * radius;
  for (int i = tid; i < span * span; i += kTile * kTile) {
    const int gx = x0 + i % span, gy = y0 + i / span;
    s_tile[i] = (gx >= 0 && gy >= 0 && gx < W && gy < H) ? in[frame + (size_t)gy * W + gx] : -INFINITY;
  }
  const int taps = 2 * radius + 1;
  for (int i = tid; i < taps * taps; i += kTile * kTile) {
    const int dx = i / taps - radius, dy = i % taps - radius;
    s_gd[i] = expf(-__fdiv_rn((float)(dx * dx + dy * dy), __fmul_rn(__fmul_rn(2.0f, sigmaD), sigmaD)));   // gaussD, filter.cu:201-204
  }
  __syncthreads();
  const int x = blockIdx.x * kTile + tx, y = blockIdx.y * kTile + ty;
  if (x >= W || y >= H) return;
  const float center = s_tile[(ty + radius) * span + tx + radius];
  float result = -INFINITY;
  if (center != -INFINITY) {
    float sum = 0.f, sumw = 0.f;
    const double denom = __dmul_rn(__dmul_rn(2.0, (double)sigmaR), (double)sigmaR);
    for (int m = 0; m < taps; ++m)                        // x outer, y inner: the reference's accumulation order
      for (int n = 0; n < taps; ++n) {
        const float cur = s_tile[(ty + n) * span + tx + m];
        if (cur != -INFINITY) {                           // out-of-image taps were staged as -inf: same skip as the bounds test
          const float dd = __fsub_rn(cur, center);
          const float gr = (float)exp(__ddiv_rn((double)(-__fmul_rn(dd, dd)), denom));       // gaussR, filter.cu:191-194
          const float w = __fmul_rn(s_gd[m * taps + n], gr);
          sumw = __fadd_rn(sumw, w);
          sum = __fmaf_rn(w, cur, sum);
        }
      }
    if (sumw > 0.f) result = __fdiv_rn(sum, sumw);
  }
  out[frame + (size_t)y * W + x] = result;
}

int launch_filter(const float* d_in, float* d_out, int W, int H, int n, float sd, float sr, cudaStream_t st) {
  const int radius = (int)ceil(2.0 * (double)sd);
  if (radius < 0 || radius > kMaxRadius) return scn::fail(SCN_ERR_ARG, "bilateral radius %d out of range (sigmaD %.3f)", radius, sd);
  dim3 grid((W + kTile - 1) / kTile, (H + kTile - 1) / kTile, n), block(kTile, kTile);
  k_bilateral<<<grid, block, 0, st>>>(d_in, d_out, W, H, sd, sr, radius);
  return SCN_OK;
}

}  // namespace

// used by run_batch (tsdf.cu) when params.depth_filter is set: u16 -> metres(-inf) -> bilateral, on the allocation stream
int scn_filter_batch(scn_tsdf* t, int n, const uint16_t* d_depth, const BatchParams& bp, int parity, const float** out) {
  const size_t px = (size_t)t->p.width * t->p.height, K = t->p.batch_frames;
  if (!t->filt_raw.p) SCN_ALLOC(t->filt_raw, 2 * K * px * 4);
  if (!t->filt_out.p) SCN_ALLOC(t->filt_out, 2 * K * px * 4);
  float* raw = t->filt_raw.as<float>() + (size_t)parity * K * px;
  float* flt = t->filt_out.as<float>() + (size_t)parity * K * px;
  dim3 g((unsigned)((px + 255) / 256), n);
  k_depth_to_metres_minf<<<g, 256, 0, t->alloc_stream.get()>>>(d_depth, bp, t->vp.depth_shift, px, raw);
  int rc = launch_filter(raw, flt, (int)t->p.width, (int)t->p.height, n, t->p.depth_sigma_d, t->p.depth_sigma_r, t->alloc_stream.get());
  if (rc) return rc;
  t->launches += 2;
  *out = flt;
  return SCN_OK;
}

// one frame of device depth -> metres (-inf invalid), bilateral-filtered into d_out when `filter` (d_raw is scratch), on `st`
int scn_depth_to_metres_device(const uint16_t* d_depth, int W, int H, float depth_shift, bool filter, float sd, float sr, float* d_raw,
                               float* d_out, cudaStream_t st) {
  const size_t px = (size_t)W * H;
  BatchParams bp; bp.n = 1; bp.f[0].src = 0;
  k_depth_to_metres_minf<<<dim3((unsigned)((px + 255) / 256), 1), 256, 0, st>>>(d_depth, bp, depth_shift, px, filter ? d_raw : d_out);
  return filter ? launch_filter(d_raw, d_out, W, H, 1, sd, sr, st) : SCN_OK;
}

extern "C" int scn_depth_bilateral_filter(const uint16_t* depth, uint32_t w, uint32_t h, float depth_shift, float sigma_d, float sigma_r,
                                          float* out_metres) {
  if (!depth || !out_metres || !w || !h || !(depth_shift > 0.f)) return scn::fail(SCN_ERR_ARG, "bad argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return scn::fail(SCN_ERR_CUDA, "no CUDA device");
  const size_t px = (size_t)w * h;
  scn::DBuf d_u16, d_a, d_b;
  SCN_ALLOC(d_u16, px * 2); SCN_ALLOC(d_a, px * 4); SCN_ALLOC(d_b, px * 4);
  SCN_CUDA_TRY(cudaMemcpy(d_u16.p, depth, px * 2, cudaMemcpyHostToDevice));
  BatchParams bp; bp.n = 1; bp.f[0].src = 0;
  k_depth_to_metres_minf<<<dim3((unsigned)((px + 255) / 256), 1), 256>>>(d_u16.as<uint16_t>(), bp, depth_shift, px, d_a.as<float>());
  int rc = launch_filter(d_a.as<float>(), d_b.as<float>(), (int)w, (int)h, 1, sigma_d, sigma_r, nullptr);
  if (!rc) { cudaError_t e = cudaMemcpy(out_metres, d_b.p, px * 4, cudaMemcpyDeviceToHost); if (e != cudaSuccess) rc = scn::fail(SCN_ERR_CUDA, "%s", cudaGetErrorString(e)); }
  return rc;
}
