// sdw_elem.cu — the HBM-bound fp32 helper kernels of the latent-walk hot path:
//   * slerp (init latents) + lerp (text embeddings), batched over all frames of a clip
//       reference: stable_diffusion_pipeline.py:466-468, utils.py:42-66
//   * classifier-free-guidance combine + linear-multistep scheduler update (+ next model input)
//       reference: stable_diffusion_pipeline.py:414-415, 421-426
//   * latent state initialisation (latents * init_noise_sigma)  — stable_diffusion_pipeline.py:401
//   * weight packing into the GEMM kernel's K-major layout
#include "sdw_internal.h"
#include "sdw_ptx.cuh"

namespace sdw {

// ---------------------------------------------------------------------------------------------
// block-wide sum of three values (fp32), result broadcast to all threads
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void block_sum3(float& a, float& b, float& c, float* sh /* >= 3*32 */) {
  a = warp_sum(a);
  b = warp_sum(b);
  c = warp_sum(c);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (lane == 0) {
    sh[warp] = a;
    sh[32 + warp] = b;
    sh[64 + warp] = c;
  }
  __syncthreads();
  a = (lane < nw) ? sh[lane] : 0.f;
  b = (lane < nw) ? sh[32 + lane] : 0.f;
  c = (lane < nw) ? sh[64 + lane] : 0.f;
  a = warp_sum(a);
  b = warp_sum(b);
  c = warp_sum(c);
  __syncthreads();
}

template <typename T>
__device__ __forceinline__ float ldf(const T* p, int64_t i);
template <>
__device__ __forceinline__ float ldf<__half>(const __half* p, int64_t i) {
  return __half2float(p[i]);
}
template <>
__device__ __forceinline__ float ldf<float>(const float* p, int64_t i) {
  return p[i];
}
template <typename T>
__device__ __forceinline__ void stf(T* p, int64_t i, float v);
template <>
__device__ __forceinline__ void stf<__half>(__half* p, int64_t i, float v) {
  p[i] = __float2half_rn(v);
}
template <>
__device__ __forceinline__ void stf<float>(float* p, int64_t i, float v) {
  p[i] = v;
}

// one block per frame: recompute the (frame-independent) dot / norms in fp32 with a fixed reduction order,
// derive the slerp weights for this frame's t, write the slerp-ed latents and the lerp-ed embeddings.
template <typename T>
__global__ void __launch_bounds__(512) slerp_lerp_kernel(const T* __restrict__ la, const T* __restrict__ lb,
                                                         const T* __restrict__ ea, const T* __restrict__ eb,
                                                         const float* __restrict__ tarr, int64_t n_lat,
                                                         int64_t n_emb, float dot_threshold, T* __restrict__ out_lat,
                                                         T* __restrict__ out_emb) {
  __shared__ float sh[96];
  const int f = blockIdx.x;
  const float t = tarr[f];
  float dab = 0.f, daa = 0.f, dbb = 0.f;
  for (int64_t i = threadIdx.x; i < n_lat; i += blockDim.x) {
    const float a = ldf(la, i), b = ldf(lb, i);
    dab = fmaf(a, b, dab);
    daa = fmaf(a, a, daa);
    dbb = fmaf(b, b, dbb);
  }
  block_sum3(dab, daa, dbb, sh);
  const float dot = dab / (sqrtf(daa) * sqrtf(dbb));
  float s0, s1;
  if (fabsf(dot) > dot_threshold) {  // utils.py:51-52 — nearly colinear: plain lerp
    s0 = 1.f - t;
    s1 = t;
  } else {  // utils.py:54-60
    const float theta0 = acosf(dot);
    const float sin0 = sinf(theta0);
    const float thetat = theta0 * t;
    s0 = sinf(theta0 - thetat) / sin0;
    s1 = sinf(thetat) / sin0;
  }
  T* ol = out_lat + static_cast<int64_t>(f) * n_lat;
  for (int64_t i = threadIdx.x; i < n_lat; i += blockDim.x) stf(ol, i, s0 * ldf(la, i) + s1 * ldf(lb, i));
  // torch.lerp(a, b, w): w < 0.5 ? a + w (b - a) : b - (b - a)(1 - w)
  T* oe = out_emb + static_cast<int64_t>(f) * n_emb;
  for (int64_t i = threadIdx.x; i < n_emb; i += blockDim.x) {
    const float a = ldf(ea, i), b = ldf(eb, i);
    const float d = b - a;
    stf(oe, i, t < 0.5f ? fmaf(t, d, a) : b - d * (1.f - t));
  }
}

int slerp_lerp_batch(const void* lat_a, const void* lat_b, const void* emb_a, const void* emb_b, const float* t,
                     int n_frames, int64_t n_lat, int64_t n_emb, int is_f16, float thr, void* out_lat, void* out_emb,
                     cudaStream_t stream) {
  SDW_REQUIRE(n_frames >= 0 && n_lat > 0 && n_emb >= 0, "bad sizes");
  if (n_frames == 0) return 0;
  SDW_REQUIRE(lat_a && lat_b && t && out_lat, "null pointer");
  if (is_f16)
    slerp_lerp_kernel<__half><<<n_frames, 512, 0, stream>>>(
        static_cast<const __half*>(lat_a), static_cast<const __half*>(lat_b), static_cast<const __half*>(emb_a),
        static_cast<const __half*>(emb_b), t, n_lat, n_emb, thr, static_cast<__half*>(out_lat),
        static_cast<__half*>(out_emb));
  else
    slerp_lerp_kernel<float><<<n_frames, 512, 0, stream>>>(
        static_cast<const float*>(lat_a), static_cast<const float*>(lat_b), static_cast<const float*>(emb_a),
        static_cast<const float*>(emb_b), t, n_lat, n_emb, thr, static_cast<float*>(out_lat),
        static_cast<float*>(out_emb));
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// CFG + scheduler step.  One thread per latent element (f, c, y, x); all arithmetic fp32.
// ---------------------------------------------------------------------------------------------
struct StepCoef {
  float guidance, c_x, c_e[5];
  int hist_slot[4];
  int use_x_base, save_x_base, push_slot;
  float next_in_scale;
  float push_e, push_x;  // hist[push_slot] := push_e * e + push_x * sample   (eps history: 1, 0; DPM-Solver++ keeps x0)
};

__global__ void cfg_sched_step_kernel(const float* __restrict__ eps, int has_uncond, float* __restrict__ x,
                                      float* __restrict__ x_base, float* __restrict__ hist, StepCoef k, int F, int C,
                                      int H, int W, __half* __restrict__ next_in, int cpad) {
  const int64_t n = static_cast<int64_t>(F) * C * H * W;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int xw = static_cast<int>(i % W);
  const int yh = static_cast<int>((i / W) % H);
  const int c = static_cast<int>((i / (static_cast<int64_t>(W) * H)) % C);
  const int f = static_cast<int>(i / (static_cast<int64_t>(W) * H * C));
  const int64_t pix = (static_cast<int64_t>(f) * H + yh) * W + xw;
  float e;
  if (has_uncond) {
    const float eu = eps[pix * C + c];
    const float ec = eps[(pix + static_cast<int64_t>(F) * H * W) * C + c];
    e = eu + k.guidance * (ec - eu);  // stable_diffusion_pipeline.py:423
  } else {
    e = eps[pix * C + c];
  }
  float xs = x[i];
  if (k.save_x_base) x_base[i] = xs;
  if (k.use_x_base) xs = x_base[i];
  float acc = k.c_e[0] * e;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (k.c_e[j + 1] != 0.f) acc = fmaf(k.c_e[j + 1], hist[static_cast<int64_t>(k.hist_slot[j]) * n + i], acc);
  const float xn = fmaf(k.c_x, xs, acc);
  if (k.push_slot >= 0) hist[static_cast<int64_t>(k.push_slot) * n + i] = fmaf(k.push_x, xs, k.push_e * e);
  x[i] = xn;
  if (next_in) {
    const __half v = __float2half_rn(xn * k.next_in_scale);
    next_in[pix * cpad + c] = v;
    if (has_uncond) next_in[(pix + static_cast<int64_t>(F) * H * W) * cpad + c] = v;
  }
}

int cfg_sched_step(const float* eps, int has_uncond, float* x, float* x_base, float* hist, const void* coef, int F,
                   int C, int H, int W, void* next_in, int cpad, cudaStream_t stream) {
  SDW_REQUIRE(eps && x && x_base && hist && coef, "null pointer");
  SDW_REQUIRE(F > 0 && C > 0 && H > 0 && W > 0, "bad sizes");
  StepCoef k;
  memcpy(&k, coef, sizeof(k));
  for (int j = 0; j < 4; ++j) SDW_REQUIRE(k.hist_slot[j] >= 0 && k.hist_slot[j] < 4, "hist slot out of range");
  SDW_REQUIRE(k.push_slot < 4, "push slot out of range");
  const int64_t n = static_cast<int64_t>(F) * C * H * W;
  const int threads = 256;
  cfg_sched_step_kernel<<<static_cast<unsigned>((n + threads - 1) / threads), threads, 0, stream>>>(
      eps, has_uncond, x, x_base, hist, k, F, C, H, W, static_cast<__half*>(next_in), cpad);
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

template <typename T>
__global__ void latents_init_kernel(const T* __restrict__ lat, float sigma, float in_scale, float* __restrict__ x,
                                    __half* __restrict__ model_in, int cpad, int dup, int F, int C, int H, int W) {
  const int64_t n = static_cast<int64_t>(F) * C * H * W;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int xw = static_cast<int>(i % W);
  const int yh = static_cast<int>((i / W) % H);
  const int c = static_cast<int>((i / (static_cast<int64_t>(W) * H)) % C);
  const int f = static_cast<int>(i / (static_cast<int64_t>(W) * H * C));
  const int64_t pix = (static_cast<int64_t>(f) * H + yh) * W + xw;
  const float v = ldf(lat, i) * sigma;  // stable_diffusion_pipeline.py:401
  x[i] = v;
  if (model_in) {
    const __half h = __float2half_rn(v * in_scale);
    model_in[pix * cpad + c] = h;
    if (dup) model_in[(pix + static_cast<int64_t>(F) * H * W) * cpad + c] = h;
  }
}

int latents_init(const void* latents, int is_f16, float sigma, float in_scale, float* x, void* model_in, int cpad,
                 int dup, int F, int C, int H, int W, cudaStream_t stream) {
  SDW_REQUIRE(latents && x, "null pointer");
  const int64_t n = static_cast<int64_t>(F) * C * H * W;
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((n + threads - 1) / threads);
  if (is_f16)
    latents_init_kernel<__half><<<blocks, threads, 0, stream>>>(static_cast<const __half*>(latents), sigma, in_scale,
                                                                 x, static_cast<__half*>(model_in), cpad, dup, F, C,
                                                                 H, W);
  else
    latents_init_kernel<float><<<blocks, threads, 0, stream>>>(static_cast<const float*>(latents), sigma, in_scale, x,
                                                                static_cast<__half*>(model_in), cpad, dup, F, C, H,
                                                                W);
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// weight packing: OIHW fp16 -> [N][kh*kw][Cp] (Cp = ceil64(C), zero padded), optional GEGLU row interleave
// ---------------------------------------------------------------------------------------------
__global__ void pack_weight_kernel(const __half* __restrict__ w, int N, int C, int taps, int Cp, int geglu,
                                   __half* __restrict__ out) {
  const int64_t total = static_cast<int64_t>(N) * taps * Cp;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % Cp);
    const int tap = static_cast<int>((i / Cp) % taps);
    const int r = static_cast<int>(i / (static_cast<int64_t>(Cp) * taps));
    int src = r;
    if (geglu) {  // packed rows: [32 value | 32 gate] per 64-row block
      const int blk = r >> 6, within = r & 63;
      src = within < 32 ? blk * 32 + within : N / 2 + blk * 32 + (within - 32);
    }
    out[i] = c < C ? w[(static_cast<int64_t>(src) * C + c) * taps + tap] : __float2half(0.f);
  }
}

// nearest-neighbour x2 upsampling followed by a 3x3 conv == four 2x2 convs on the LOW-res grid, one per output
// parity (py, px): the taps that read the same low-res pixel are pre-summed (fp32, rounded once to fp16), which cuts
// the upsampler FLOPs by 9/4.  Layout per parity: [N][4 taps (a*2+b)][Cp]; row group a / column group b:
//   parity 0: group 0 = {k=0} (shift -1), group 1 = {k=1,2} (shift 0);  parity 1: group 0 = {k=0,1} (0), group 1 = {k=2} (+1)
__global__ void pack_weight_up4_kernel(const __half* __restrict__ w, int N, int C, int Cp, __half* __restrict__ out) {
  const int64_t per = static_cast<int64_t>(N) * 4 * Cp;
  const int64_t total = per * 4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int par = static_cast<int>(i / per);
    const int64_t r = i - par * per;
    const int c = static_cast<int>(r % Cp);
    const int tap = static_cast<int>((r / Cp) % 4);
    const int n = static_cast<int>(r / (static_cast<int64_t>(Cp) * 4));
    const int py = par >> 1, px = par & 1, a = tap >> 1, b = tap & 1;
    float acc = 0.f;
    if (c < C) {
      const int ky0 = py == 0 ? (a == 0 ? 0 : 1) : (a == 0 ? 0 : 2);
      const int ky1 = py == 0 ? (a == 0 ? 0 : 2) : (a == 0 ? 1 : 2);
      const int kx0 = px == 0 ? (b == 0 ? 0 : 1) : (b == 0 ? 0 : 2);
      const int kx1 = px == 0 ? (b == 0 ? 0 : 2) : (b == 0 ? 1 : 2);
      for (int ky = ky0; ky <= ky1; ++ky)
        for (int kx = kx0; kx <= kx1; ++kx) acc += __half2float(w[((static_cast<int64_t>(n) * C + c) * 3 + ky) * 3 + kx]);
    }
    out[i] = __float2half_rn(acc);
  }
}

int pack_weight_up4(const void* w, int N, int C, void* out, cudaStream_t stream) {
  SDW_REQUIRE(w && out && N > 0 && C > 0, "bad weight");
  const int Cp = (C + 63) / 64 * 64;
  const int64_t total = static_cast<int64_t>(N) * 16 * Cp;
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((total + 255) / 256, static_cast<int64_t>(sm_count()) * 16));
  pack_weight_up4_kernel<<<blocks, 256, 0, stream>>>(static_cast<const __half*>(w), N, C, Cp, static_cast<__half*>(out));
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

int pack_weight(const void* w, int N, int C, int kh, int kw, int geglu, void* out, cudaStream_t stream) {
  SDW_REQUIRE(w && out && N > 0 && C > 0 && kh > 0 && kw > 0, "bad weight");
  if (geglu) SDW_REQUIRE(N % 64 == 0, "GEGLU interleave needs N % 64 == 0");
  const int Cp = (C + 63) / 64 * 64;
  const int64_t total = static_cast<int64_t>(N) * kh * kw * Cp;
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((total + threads - 1) / threads, static_cast<int64_t>(sm_count()) * 16));
  pack_weight_kernel<<<blocks, threads, 0, stream>>>(static_cast<const __half*>(w), N, C, kh * kw, Cp, geglu,
                                                     static_cast<__half*>(out));
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}


// ---------------------------------------------------------------------------------------------
// tiled = True (stable_diffusion_pipeline.py:841-858: every Conv2d gets padding_mode="circular"): a padded convolution on
// the torus is a zero-padded convolution of the wrap-padded image, cropped.  wrap_pad copies an NHWC image into a dense
// (H + 2 pad) x (W + 2 pad) one whose border repeats the opposite edge; crop takes the interior of the padded result back
// out (adding a residual for the fp16 case).  Element size is generic (fp16 activations, fp32 eps, uint8 frames).
// ---------------------------------------------------------------------------------------------
template <int VEC>
__global__ void wrap_pad_kernel(const uint8_t* __restrict__ x, int64_t ld_bytes, int B, int H, int W, int pix_bytes, int pad,
                                uint8_t* __restrict__ y) {
  const int Hp = H + 2 * pad, Wp = W + 2 * pad, chunks = pix_bytes / VEC;
  const int64_t n = static_cast<int64_t>(B) * Hp * Wp * chunks;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = static_cast<int>(i % chunks);
  const int64_t pp = i / chunks;
  const int xp = static_cast<int>(pp % Wp), yp = static_cast<int>((pp / Wp) % Hp);
  const int64_t b = pp / (static_cast<int64_t>(Wp) * Hp);
  const int xs = ((xp - pad) % W + W) % W, ys = ((yp - pad) % H + H) % H;
  const uint8_t* src = x + ((b * H + ys) * W + xs) * ld_bytes + static_cast<int64_t>(c) * VEC;
  uint8_t* dst = y + pp * pix_bytes + static_cast<int64_t>(c) * VEC;
  if (VEC == 16) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
  else if (VEC == 8) *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(src);
  else *dst = *src;
}

template <int VEC>
__global__ void crop_kernel(const uint8_t* __restrict__ yp, int B, int H, int W, int pix_bytes, int crop,
                            const __half* __restrict__ resid, int64_t ldr, uint8_t* __restrict__ out, int64_t ldo_bytes) {
  const int Wp = W + 2 * crop, Hp = H + 2 * crop, chunks = pix_bytes / VEC;
  const int64_t n = static_cast<int64_t>(B) * H * W * chunks;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = static_cast<int>(i % chunks);
  const int64_t p = i / chunks;
  const int xw = static_cast<int>(p % W), yh = static_cast<int>((p / W) % H);
  const int64_t b = p / (static_cast<int64_t>(W) * H);
  const uint8_t* src = yp + ((b * Hp + yh + crop) * Wp + xw + crop) * pix_bytes + static_cast<int64_t>(c) * VEC;
  uint8_t* dst = out + p * ldo_bytes + static_cast<int64_t>(c) * VEC;
  if (VEC == 16) {
    uint4 v = *reinterpret_cast<const uint4*>(src);
    if (resid) {
      const uint4 r = *reinterpret_cast<const uint4*>(resid + p * ldr + c * 8);
      __half2* a = reinterpret_cast<__half2*>(&v);
      const __half2* q = reinterpret_cast<const __half2*>(&r);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 fa = __half22float2(a[k]), fb = __half22float2(q[k]);
        a[k] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
      }
    }
    *reinterpret_cast<uint4*>(dst) = v;
  } else if (VEC == 8) {
    *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(src);
  } else {
    *dst = *src;
  }
}

int wrap_pad(const void* x, int64_t ld_bytes, int B, int H, int W, int pix_bytes, int pad, void* y, cudaStream_t stream) {
  SDW_REQUIRE(x && y && B > 0 && H > 0 && W > 0 && pix_bytes > 0 && pad >= 1 && pad <= H && pad <= W, "wrap_pad: bad arguments");
  const int vec = (pix_bytes % 16 == 0 && ld_bytes % 16 == 0) ? 16 : ((pix_bytes % 8 == 0 && ld_bytes % 8 == 0) ? 8 : 1);
  const int64_t n = static_cast<int64_t>(B) * (H + 2 * pad) * (W + 2 * pad) * (pix_bytes / vec);
  const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
  const uint8_t* xs = static_cast<const uint8_t*>(x);
  uint8_t* ys = static_cast<uint8_t*>(y);
  if (vec == 16) wrap_pad_kernel<16><<<blocks, 256, 0, stream>>>(xs, ld_bytes, B, H, W, pix_bytes, pad, ys);
  else if (vec == 8) wrap_pad_kernel<8><<<blocks, 256, 0, stream>>>(xs, ld_bytes, B, H, W, pix_bytes, pad, ys);
  else wrap_pad_kernel<1><<<blocks, 256, 0, stream>>>(xs, ld_bytes, B, H, W, pix_bytes, pad, ys);
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

int crop_interior(const void* yp, int B, int H, int W, int pix_bytes, int crop, const void* resid_f16, int64_t ldr, void* out,
                  int64_t ldo_bytes, cudaStream_t stream) {
  SDW_REQUIRE(yp && out && B > 0 && H > 0 && W > 0 && pix_bytes > 0 && crop >= 1, "crop: bad arguments");
  const int vec = (pix_bytes % 16 == 0 && ldo_bytes % 16 == 0) ? 16 : ((pix_bytes % 8 == 0 && ldo_bytes % 8 == 0) ? 8 : 1);
  SDW_REQUIRE(!resid_f16 || (vec == 16 && ldr % 8 == 0), "crop: the residual add needs 16-byte channel chunks");
  const int64_t n = static_cast<int64_t>(B) * H * W * (pix_bytes / vec);
  const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
  const uint8_t* ys = static_cast<const uint8_t*>(yp);
  const __half* rs = static_cast<const __half*>(resid_f16);
  uint8_t* os = static_cast<uint8_t*>(out);
  if (vec == 16) crop_kernel<16><<<blocks, 256, 0, stream>>>(ys, B, H, W, pix_bytes, crop, rs, ldr, os, ldo_bytes);
  else if (vec == 8) crop_kernel<8><<<blocks, 256, 0, stream>>>(ys, B, H, W, pix_bytes, crop, nullptr, 0, os, ldo_bytes);
  else crop_kernel<1><<<blocks, 256, 0, stream>>>(ys, B, H, W, pix_bytes, crop, nullptr, 0, os, ldo_bytes);
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sdw
