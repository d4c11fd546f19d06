// sdw_safety.cu — the Stable Diffusion safety checker behind `__call__`'s post-decode filter
// (stable_diffusion_pipeline.py:440-447), natively: CLIPFeatureExtractor preprocessing (Pillow bicubic resize of the
// shortest edge to 224, centre crop, CLIP normalisation), the CLIP ViT image tower, the visual projection and the
// diffusers concept-score loop, which flags frames and (optionally) blacks them out on the device.
//
// Preprocessing is bit-exact with Pillow at the uint8 stage: the host builds Pillow's coefficient tables
// (precompute_coeffs + normalize_coeffs_8bpc, 22-bit fixed point) and two kernels run its horizontal-then-vertical
// passes, the vertical one only for the 224 x 224 pixels the crop keeps.  The patch conv is a GEMM whose A rows are
// written by the normalisation kernel; the transformer layers are the CLIP text tower's `ClipEncoder` (sdw_clip.cu)
// without the causal mask: the QKV GEMM with the V^T epilogue and the sampler's fused attention.  State-dict names are
// diffusers' `StableDiffusionSafetyChecker` keys.
#include "sdw_internal.h"
#include "sdw_ptx.cuh"

#include <cmath>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/sdwalk.h"

namespace sdw {

constexpr int SAFETY_CROP = 224;
constexpr int SAFETY_MAX_SCORES = 64;  // special + regular concepts the score kernel stages

// ---------------------------------------------------------------------------------------------
// host: Pillow's resampling coefficients (libImaging/Resample.c), restated for the bicubic filter
// ---------------------------------------------------------------------------------------------
static double pil_bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// coefficients of output samples first .. first + count - 1 of an in_size -> out_size resize, as int32 with 22
// fractional bits (rounded away from zero); bounds[2i] = first input sample, bounds[2i + 1] = taps; returns ksize
static int pil_coeffs(int in_size, int out_size, int first, int count, std::vector<int32_t>& kk, std::vector<int32_t>& bounds) {
  const double scale = static_cast<double>(static_cast<float>(in_size) - 0.f) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * filterscale;
  const int ksize = static_cast<int>(std::ceil(support)) * 2 + 1;
  kk.assign(static_cast<size_t>(count) * ksize, 0);
  bounds.assign(static_cast<size_t>(count) * 2, 0);
  std::vector<double> k(ksize);
  for (int i = 0; i < count; ++i) {
    const int xx = first + i;
    const double center = (xx + 0.5) * scale;
    const double ss = 1.0 / filterscale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      const double w = pil_bicubic((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    for (int x = 0; x < xmax; ++x) {
      if (ww != 0.0) k[x] /= ww;
      const double v = k[x] * (1 << 22);
      kk[static_cast<size_t>(i) * ksize + x] = v < 0 ? static_cast<int32_t>(-0.5 + v) : static_cast<int32_t>(0.5 + v);
    }
    bounds[2 * i] = xmin;
    bounds[2 * i + 1] = xmax;
  }
  return ksize;
}

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t pil_clip8(int v) {
  if (v >= (1 << 30)) return 255;
  if (v <= 0) return 0;
  return static_cast<uint8_t>(v >> 22);
}

// horizontal pass: src [B][H][W][3] -> tmp [B][H][224][3] (the 224 crop columns of the resized width)
__global__ void safety_hresize_kernel(const uint8_t* __restrict__ src, int H, int W, const int32_t* __restrict__ kk,
                                      const int32_t* __restrict__ bounds, int ksize, uint8_t* __restrict__ tmp) {
  const int j = threadIdx.x, y = blockIdx.x, b = blockIdx.y;
  const int xmin = bounds[2 * j], xn = bounds[2 * j + 1];
  const int32_t* k = kk + static_cast<int64_t>(j) * ksize;
  const uint8_t* row = src + ((static_cast<int64_t>(b) * H + y) * W + xmin) * 3;
  int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
  for (int x = 0; x < xn; ++x) {
    s0 += row[3 * x] * k[x];
    s1 += row[3 * x + 1] * k[x];
    s2 += row[3 * x + 2] * k[x];
  }
  uint8_t* o = tmp + ((static_cast<int64_t>(b) * H + y) * SAFETY_CROP + j) * 3;
  o[0] = pil_clip8(s0);
  o[1] = pil_clip8(s1);
  o[2] = pil_clip8(s2);
}

// vertical pass over the 224 crop rows: tmp [B][H][224][3] -> crop [B][224][224][3]
__global__ void safety_vresize_kernel(const uint8_t* __restrict__ tmp, int H, const int32_t* __restrict__ kk,
                                      const int32_t* __restrict__ bounds, int ksize, uint8_t* __restrict__ crop) {
  const int j = threadIdx.x, i = blockIdx.x, b = blockIdx.y;
  const int ymin = bounds[2 * i], yn = bounds[2 * i + 1];
  const int32_t* k = kk + static_cast<int64_t>(i) * ksize;
  const uint8_t* col = tmp + ((static_cast<int64_t>(b) * H + ymin) * SAFETY_CROP + j) * 3;
  int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
  for (int y = 0; y < yn; ++y) {
    const uint8_t* p = col + static_cast<int64_t>(y) * SAFETY_CROP * 3;
    s0 += p[0] * k[y];
    s1 += p[1] * k[y];
    s2 += p[2] * k[y];
  }
  uint8_t* o = crop + ((static_cast<int64_t>(b) * SAFETY_CROP + i) * SAFETY_CROP + j) * 3;
  o[0] = pil_clip8(s0);
  o[1] = pil_clip8(s1);
  o[2] = pil_clip8(s2);
}

struct Norm3 {
  float mean[3], std[3];
};

// (u / 255 - mean) / std rounded to fp16 once, written as patch GEMM rows a [B * np][Kp] in (c, ky, kx) order with the
// columns K .. Kp - 1 zero; blocks past B * np write the class tokens x[b][0] = class + pos[0].  pix (optional) receives
// the normalised image [B][224][224][3].
__global__ void safety_patchify_kernel(const uint8_t* __restrict__ crop, int B, int patch, int Kp, Norm3 nm,
                                       __half* __restrict__ a, __half* __restrict__ pix, const __half* __restrict__ cls,
                                       const __half* __restrict__ pos, int hidden, int ntok, __half* __restrict__ x) {
  const int per_row = SAFETY_CROP / patch, np = per_row * per_row;
  const int row = blockIdx.x;
  if (row >= B * np) {
    const int b = row - B * np;
    __half* o = x + static_cast<int64_t>(b) * ntok * hidden;
    for (int i = threadIdx.x; i < hidden; i += blockDim.x)
      o[i] = __float2half_rn(__half2float(cls[i]) + __half2float(pos[i]));
    return;
  }
  const int b = row / np, pi = row % np, py = pi / per_row, px = pi % per_row;
  const int pp = patch * patch, K = 3 * pp;
  for (int k = threadIdx.x; k < Kp; k += blockDim.x) {
    __half v = __float2half_rn(0.f);
    if (k < K) {
      const int c = k / pp, r = k % pp, y = py * patch + r / patch, xx = px * patch + r % patch;
      const int64_t off = ((static_cast<int64_t>(b) * SAFETY_CROP + y) * SAFETY_CROP + xx) * 3 + c;
      v = __float2half_rn((static_cast<float>(crop[off]) / 255.f - nm.mean[c]) / nm.std[c]);
      if (pix) pix[off] = v;
    }
    a[static_cast<int64_t>(row) * Kp + k] = v;
  }
}

__device__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) t += red[w];
  return t;
}

// One block per image: fp32 cosines of the image embedding against the special-care and concept embeddings, then the
// diffusers decision loop in fp64 (NumPy-1.x promotion of float32 - float), each score rounded to 3 decimals as
// np.round does (rint(x * 1000) / 1000, half to even).  A flagged frame is zeroed in place when `frames` is given.
__global__ void __launch_bounds__(256) safety_score_kernel(const float* __restrict__ emb, int D,
                                                           const float* __restrict__ special,
                                                           const float* __restrict__ special_w, int ns,
                                                           const float* __restrict__ concepts,
                                                           const float* __restrict__ concept_w, int nc,
                                                           int32_t* __restrict__ flags, float* __restrict__ cos_out,
                                                           double* __restrict__ score_out, uint8_t* __restrict__ frames,
                                                           int64_t frame_bytes) {
  __shared__ float red[32];
  __shared__ float cs[SAFETY_MAX_SCORES];
  __shared__ int flagged;
  const int b = blockIdx.x;
  const float* e = emb + static_cast<int64_t>(b) * D;
  float ee = 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) ee = fmaf(e[i], e[i], ee);
  ee = block_sum(ee, red);
  const float en = fmaxf(sqrtf(ee), 1e-12f);
  for (int j = 0; j < ns + nc; ++j) {
    const float* c = j < ns ? special + static_cast<int64_t>(j) * D : concepts + static_cast<int64_t>(j - ns) * D;
    float dot = 0.f, cc = 0.f;
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      dot = fmaf(e[i], c[i], dot);
      cc = fmaf(c[i], c[i], cc);
    }
    dot = block_sum(dot, red);
    cc = block_sum(cc, red);
    if (threadIdx.x == 0) cs[j] = dot / (en * fmaxf(sqrtf(cc), 1e-12f));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double adjustment = 0.0;
    int bad = 0;
    for (int j = 0; j < ns + nc; ++j) {
      const double thr = j < ns ? static_cast<double>(special_w[j]) : static_cast<double>(concept_w[j - ns]);
      const double s = rint((static_cast<double>(cs[j]) - thr + adjustment) * 1000.0) / 1000.0;
      if (j < ns) {
        if (s > 0) adjustment = 0.01;
      } else if (s > 0) {
        bad = 1;
      }
      if (cos_out) cos_out[static_cast<int64_t>(b) * (ns + nc) + j] = cs[j];
      if (score_out) score_out[static_cast<int64_t>(b) * (ns + nc) + j] = s;
    }
    flags[b] = bad;
    flagged = bad;
  }
  __syncthreads();
  if (frames && flagged) {
    uint8_t* f = frames + static_cast<int64_t>(b) * frame_bytes;
    for (int64_t i = threadIdx.x; i < frame_bytes; i += blockDim.x) f[i] = 0;
  }
}

// ---------------------------------------------------------------------------------------------
// engine
// ---------------------------------------------------------------------------------------------
struct SafetyTower {  // the transformer ops of one chunk size, replayed as a CUDA graph
  OpList ops;
  GraphCache graph;
};

struct SafetyEngine {
  sdw_safety_config cfg;
  Arena arena{256};
  size_t cap = 0;
  ParamTable params;
  ClipEncoder enc;
  int np = 0, ntok = 0, K = 0, Kp = 0;
  int64_t vt_ld = 0;
  __half *patch_w = nullptr, *cls = nullptr, *pos = nullptr, *proj_w = nullptr;
  float *pre_g = nullptr, *pre_b = nullptr, *post_g = nullptr, *post_b = nullptr;
  float *special = nullptr, *special_w = nullptr, *concepts = nullptr, *concept_w = nullptr;
  __half *a = nullptr, *x0 = nullptr, *x1 = nullptr, *h = nullptr, *qk = nullptr, *vt = nullptr, *ff = nullptr,
         *pooled = nullptr;
  float *pooled32 = nullptr, *embeds = nullptr;
  uint8_t* crop = nullptr;
  std::map<int, std::unique_ptr<SafetyTower>> towers;
  // resize tables and the horizontal-pass buffer of the current frame size, for chunks of max_batch frames (device
  // memory owned here: its size depends on the frame height, which the arena is not sized for)
  int rs_H = 0, rs_W = 0, kh = 0, kv = 0;
  void* rs_mem = nullptr;
  int32_t *hk = nullptr, *hb = nullptr, *vk = nullptr, *vb = nullptr;
  uint8_t* tmp = nullptr;

  ~SafetyEngine() {
    if (rs_mem) cudaFree(rs_mem);
  }

  void layout(void* base) {
    const sdw_safety_config& c = cfg;
    const int Hd = c.hidden, I = c.intermediate;
    np = (c.image_size / c.patch) * (c.image_size / c.patch);
    ntok = np + 1;
    K = 3 * c.patch * c.patch;
    Kp = (K + 63) / 64 * 64;
    vt_ld = (ntok + 7) / 8 * 8;
    arena.reset(base);
    params.clear(base != nullptr);
    towers.clear();
    const std::string vm = "vision_model.vision_model.";
    cls = arena.take<__half>(Hd);
    patch_w = arena.take<__half>(static_cast<size_t>(Hd) * Kp);
    pos = arena.take<__half>(static_cast<size_t>(ntok) * Hd);
    params.add(vm + "embeddings.class_embedding", RAW, cls, Hd);
    params.add(vm + "embeddings.patch_embedding.weight", PACKED, patch_w, static_cast<int64_t>(Hd) * K, Hd, K);
    params.add(vm + "embeddings.position_embedding.weight", RAW, pos, static_cast<int64_t>(ntok) * Hd);
    pre_g = arena.take<float>(Hd); pre_b = arena.take<float>(Hd);
    params.add(vm + "pre_layrnorm.weight", VEC, pre_g, Hd);
    params.add(vm + "pre_layrnorm.bias", VEC, pre_b, Hd);
    enc.layout(arena, params, vm + "encoder.layers.", c.layers, Hd, I);
    post_g = arena.take<float>(Hd); post_b = arena.take<float>(Hd);
    params.add(vm + "post_layernorm.weight", VEC, post_g, Hd);
    params.add(vm + "post_layernorm.bias", VEC, post_b, Hd);
    proj_w = arena.take<__half>(static_cast<size_t>(c.proj_dim) * Hd);
    params.add("visual_projection.weight", RAW, proj_w, static_cast<int64_t>(c.proj_dim) * Hd);
    concepts = arena.take<float>(static_cast<size_t>(c.n_concepts) * c.proj_dim);
    special = arena.take<float>(static_cast<size_t>(c.n_special) * c.proj_dim);
    concept_w = arena.take<float>(c.n_concepts);
    special_w = arena.take<float>(c.n_special);
    params.add("concept_embeds", VEC, concepts, static_cast<int64_t>(c.n_concepts) * c.proj_dim);
    params.add("special_care_embeds", VEC, special, static_cast<int64_t>(c.n_special) * c.proj_dim);
    params.add("concept_embeds_weights", VEC, concept_w, c.n_concepts);
    params.add("special_care_embeds_weights", VEC, special_w, c.n_special);
    const size_t mb = c.max_batch, T = mb * ntok;
    a = arena.take<__half>(mb * np * Kp);
    x0 = arena.take<__half>(T * Hd); x1 = arena.take<__half>(T * Hd); h = arena.take<__half>(T * Hd);
    qk = arena.take<__half>(T * 2 * Hd);
    vt = arena.take<__half>(mb * Hd * vt_ld);
    ff = arena.take<__half>(T * I);
    pooled = arena.take<__half>(mb * Hd);
    pooled32 = arena.take<float>(mb * Hd);
    embeds = arena.take<float>(mb * c.proj_dim);
    crop = arena.take<uint8_t>(mb * SAFETY_CROP * SAFETY_CROP * 3);
  }

  // patch GEMM .. image embeddings for a chunk of B images whose patch rows and class tokens are in place
  int build_tower(int B, SafetyTower& t) {
    const sdw_safety_config& c = cfg;
    const int Hd = c.hidden;
    const int64_t T = static_cast<int64_t>(B) * ntok;
    OpList& ops = t.ops;
    ops.clear();
    {
      GemmDesc d;  // tokens 1..np of every sample, + pos[1..np] broadcast over the samples
      d.A = a; d.C = K; d.W = np; d.H = 1; d.B = B; d.sW = Kp; d.sB = static_cast<int64_t>(np) * Kp;
      d.Wt = patch_w; d.N = Hd;
      d.out = x0 + Hd; d.o_sW = Hd; d.o_sB = static_cast<int64_t>(ntok) * Hd;
      d.resid = pos + Hd; d.r_sW = Hd; d.r_sB = 0;
      d.et = 1;  // the residual's batch stride 0 is not a tensor-map view
      if (int e = ops.add_gemm(d, "patch embedding " + std::to_string(K) + "->" + std::to_string(Hd) + " + pos")) return e;
    }
    const float eps = c.eps;
    ops.add("pre_layrnorm", [=](cudaStream_t st, int) { return layernorm(x0, Hd, T, Hd, pre_g, pre_b, eps, x1, Hd, st); });
    ClipEncoder::Buffers b;
    b.x = x1; b.y = x0; b.h = h; b.ff = ff; b.qkv = qk; b.vt = vt; b.vt_ld = vt_ld;
    if (int e = enc.emit(ops, B, ntok, eps, c.act, false, b)) return e;
    const int P = c.proj_dim;
    __half* pl = pooled;
    float *p32 = pooled32, *emb = embeds;
    ops.add("post_layernorm (CLS)", [=](cudaStream_t st, int) {  // the encoder's result is in x1
      return layernorm(x1, static_cast<int64_t>(ntok) * Hd, B, Hd, post_g, post_b, eps, pl, Hd, st);
    });
    ops.add("visual_projection (fp32)", [=](cudaStream_t st, int) {
      if (int rc = half_to_float(pl, p32, static_cast<int64_t>(B) * Hd, 0, 1.f, st)) return rc;
      return linear_f32(p32, Hd, proj_w, nullptr, B, P, Hd, 0, 0, emb, P, st);
    });
    return 0;
  }

  SafetyTower* tower(int B) {
    auto it = towers.find(B);
    if (it != towers.end()) return it->second.get();
    auto t = std::make_unique<SafetyTower>();
    if (build_tower(B, *t)) return nullptr;
    return (towers[B] = std::move(t)).get();
  }

  // Pillow tables and the horizontal-pass buffer for frames of H x W.  Only the first call for a frame size does work,
  // and it is synchronous: cudaFree / cudaMalloc of the buffer and the upload of the host-built tables.  A walk has
  // one frame size, so its later calls only enqueue kernels.
  int prepare(int H, int W) {
    if (rs_mem && rs_H == H && rs_W == W) return 0;
    int nh, nw;  // transformers' get_resize_output_image_size(default_to_square=False): short edge -> 224
    if (W <= H) {
      nw = SAFETY_CROP;
      nh = static_cast<int>(static_cast<double>(SAFETY_CROP) * H / W);
    } else {
      nh = SAFETY_CROP;
      nw = static_cast<int>(static_cast<double>(SAFETY_CROP) * W / H);
    }
    const int top = (nh - SAFETY_CROP) / 2, left = (nw - SAFETY_CROP) / 2;
    std::vector<int32_t> hkk, hbb, vkk, vbb;
    kh = pil_coeffs(W, nw, left, SAFETY_CROP, hkk, hbb);
    kv = pil_coeffs(H, nh, top, SAFETY_CROP, vkk, vbb);
    const size_t n_i32 = hkk.size() + hbb.size() + vkk.size() + vbb.size();
    const size_t tmp_bytes = static_cast<size_t>(cfg.max_batch) * H * SAFETY_CROP * 3;
    if (rs_mem) cudaFree(rs_mem);
    rs_mem = nullptr;
    SDW_CUDA_OK(cudaMalloc(&rs_mem, n_i32 * 4 + tmp_bytes));
    int32_t* p = static_cast<int32_t*>(rs_mem);
    hk = p; p += hkk.size();
    hb = p; p += hbb.size();
    vk = p; p += vkk.size();
    vb = p; p += vbb.size();
    tmp = reinterpret_cast<uint8_t*>(p);
    SDW_CUDA_OK(cudaMemcpy(hk, hkk.data(), hkk.size() * 4, cudaMemcpyHostToDevice));
    SDW_CUDA_OK(cudaMemcpy(hb, hbb.data(), hbb.size() * 4, cudaMemcpyHostToDevice));
    SDW_CUDA_OK(cudaMemcpy(vk, vkk.data(), vkk.size() * 4, cudaMemcpyHostToDevice));
    SDW_CUDA_OK(cudaMemcpy(vb, vbb.data(), vbb.size() * 4, cudaMemcpyHostToDevice));
    rs_H = H;
    rs_W = W;
    return 0;
  }

  // frames [B][H][W][3] -> crop (uint8), patch rows (into `rows`, the arena's A operand by default) and class tokens;
  // pix optional fp16 [B][224][224][3]
  int preprocess(const uint8_t* frames, int B, int H, int W, __half* pix, cudaStream_t st, __half* rows = nullptr) {
    safety_hresize_kernel<<<dim3(H, B), SAFETY_CROP, 0, st>>>(frames, H, W, hk, hb, kh, tmp);
    SDW_CUDA_OK(cudaGetLastError());
    safety_vresize_kernel<<<dim3(SAFETY_CROP, B), SAFETY_CROP, 0, st>>>(tmp, H, vk, vb, kv, crop);
    SDW_CUDA_OK(cudaGetLastError());
    Norm3 nm;
    for (int c = 0; c < 3; ++c) {
      nm.mean[c] = cfg.mean[c];
      nm.std[c] = cfg.std[c];
    }
    safety_patchify_kernel<<<B * np + B, 128, 0, st>>>(crop, B, cfg.patch, Kp, nm, rows ? rows : a, pix, cls, pos,
                                                       cfg.hidden, ntok, x0);
    SDW_CUDA_OK(cudaGetLastError());
    return 0;
  }

  int scores(const float* emb, int B, int32_t* flags, float* cos, double* sc, uint8_t* frames, int64_t frame_bytes,
             cudaStream_t st) {
    safety_score_kernel<<<B, 256, 0, st>>>(emb, cfg.proj_dim, special, special_w, cfg.n_special, concepts, concept_w,
                                           cfg.n_concepts, flags, cos, sc, frames, frame_bytes);
    SDW_CUDA_OK(cudaGetLastError());
    return 0;
  }

  // the whole checker over B frames in chunks of max_batch; embeds_out (optional) receives the image embeddings
  int run(const uint8_t* frames_in, uint8_t* frames_blackout, int B, int H, int W, int32_t* flags, float* cos,
          float* embeds_out, int use_graph, cudaStream_t st) {
    const int mb = cfg.max_batch;
    if (int rc = prepare(H, W)) return rc;
    const int64_t fb = static_cast<int64_t>(H) * W * 3;
    for (int i0 = 0; i0 < B; i0 += mb) {
      const int n = std::min(mb, B - i0);
      SafetyTower* t = tower(n);
      if (!t) return 1;
      if (int rc = preprocess(frames_in + i0 * fb, n, H, W, nullptr, st)) return rc;
      if (use_graph) {
        if (int rc = t->graph.launch(n, st, [t](cudaStream_t s) { return t->ops.run(s, 0); })) return rc;
      } else if (int rc = t->ops.run(st, 0)) {
        return rc;
      }
      if (embeds_out)
        SDW_CUDA_OK(cudaMemcpyAsync(embeds_out + static_cast<int64_t>(i0) * cfg.proj_dim, embeds,
                                    static_cast<size_t>(n) * cfg.proj_dim * 4, cudaMemcpyDeviceToDevice, st));
      if (flags) {
        float* c = cos ? cos + static_cast<int64_t>(i0) * (cfg.n_special + cfg.n_concepts) : nullptr;
        if (int rc = scores(embeds, n, flags + i0, c, nullptr, frames_blackout ? frames_blackout + i0 * fb : nullptr, fb, st))
          return rc;
      }
    }
    return 0;
  }
};

static int frames_ok(const SafetyEngine* E, const void* frames, int B, int H, int W) {
  SDW_REQUIRE(E && frames && E->params.bound, "null / engine not bound");
  SDW_REQUIRE(E->params.missing(nullptr) == 0, "safety checker parameters not loaded");
  SDW_REQUIRE(B >= 1 && H >= 1 && W >= 1 && H <= 16384 && W <= 16384, "safety checker: bad frame count or size");
  SDW_REQUIRE(static_cast<int64_t>(E->cfg.max_batch) * H * SAFETY_CROP * 3 < (int64_t(1) << 31),
              "safety checker: frames too tall");
  return 0;
}

}  // namespace sdw

using namespace sdw;

extern "C" {

int sdw_safety_create(const sdw_safety_config* cfg, sdw_safety** out) {
  SDW_REQUIRE(cfg && out, "null");
  SDW_REQUIRE(cfg->hidden % 64 == 0 && cfg->hidden == cfg->heads * 64, "CLIP vision towers here have 64-wide heads");
  SDW_REQUIRE(cfg->intermediate % 64 == 0 && cfg->layers >= 1, "bad CLIP vision configuration");
  SDW_REQUIRE(cfg->image_size == SAFETY_CROP, "image_size must be 224 (the feature extractor's crop)");
  SDW_REQUIRE(cfg->patch >= 1 && SAFETY_CROP % cfg->patch == 0, "patch must divide 224");
  SDW_REQUIRE(cfg->proj_dim >= 1 && cfg->proj_dim % 8 == 0, "proj_dim must be a positive multiple of 8");
  SDW_REQUIRE(cfg->n_concepts >= 0 && cfg->n_special >= 0 && cfg->n_concepts + cfg->n_special <= SAFETY_MAX_SCORES,
              "at most 64 concepts in all");
  SDW_REQUIRE(cfg->n_concepts + cfg->n_special >= 1, "no concepts");
  SDW_REQUIRE(cfg->act == 0 || cfg->act == 1, "act: 0 quick-GELU, 1 erf GELU");
  SDW_REQUIRE(cfg->max_batch >= 1 && cfg->max_batch <= 64, "max_batch in 1..64");
  SDW_REQUIRE(cfg->eps > 0.f, "eps");
  for (int c = 0; c < 3; ++c) SDW_REQUIRE(cfg->std[c] > 0.f, "std must be positive");
  SafetyEngine* E = new SafetyEngine();
  E->cfg = *cfg;
  E->layout(nullptr);
  E->cap = E->arena.off;
  *out = reinterpret_cast<sdw_safety*>(E);
  return 0;
}

void sdw_safety_destroy(sdw_safety* e) { delete reinterpret_cast<SafetyEngine*>(e); }

int sdw_safety_arena_bytes(const sdw_safety* e, uint64_t* bytes) {
  const SafetyEngine* E = reinterpret_cast<const SafetyEngine*>(e);
  SDW_REQUIRE(E && bytes, "null");
  *bytes = E->cap + 256;
  return 0;
}

int sdw_safety_bind(sdw_safety* e, void* arena, uint64_t bytes) {
  SafetyEngine* E = reinterpret_cast<SafetyEngine*>(e);
  SDW_REQUIRE(E && arena, "null");
  SDW_REQUIRE(bytes >= E->cap + 256, "arena too small");
  SDW_REQUIRE((reinterpret_cast<uintptr_t>(arena) & 255) == 0, "arena must be 256-byte aligned");
  E->layout(arena);
  return 0;
}

int sdw_safety_num_params(const sdw_safety* e) { return e ? reinterpret_cast<const SafetyEngine*>(e)->params.size() : 0; }

int sdw_safety_param_info(const sdw_safety* e, int index, const char** name, int64_t* numel) {
  SDW_REQUIRE(e, "null");
  return reinterpret_cast<const SafetyEngine*>(e)->params.info(index, name, numel);
}

int sdw_safety_load_param(sdw_safety* e, const char* name, const void* data_f16, int64_t numel, void* stream) {
  SDW_REQUIRE(e, "null");
  return reinterpret_cast<SafetyEngine*>(e)->params.load(name, data_f16, numel, static_cast<cudaStream_t>(stream));
}

int sdw_safety_missing_params(const sdw_safety* e, const char** first_missing) {
  return e ? reinterpret_cast<const SafetyEngine*>(e)->params.missing(first_missing) : -1;
}

int sdw_safety_check(sdw_safety* e, void* frames_u8, int B, int H, int W, int32_t* flags, float* cos_f32, int blackout,
                     void* stream) {
  SafetyEngine* E = reinterpret_cast<SafetyEngine*>(e);
  if (int rc = frames_ok(E, frames_u8, B, H, W)) return rc;
  SDW_REQUIRE(flags, "null flags");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDW_REQUIRE(st != nullptr, "graph capture needs a real stream, not the legacy default stream 0");
  uint8_t* f = static_cast<uint8_t*>(frames_u8);
  return E->run(f, blackout ? f : nullptr, B, H, W, flags, cos_f32, nullptr, 1, st);
}

int sdw_safety_preprocess(sdw_safety* e, const uint8_t* frames_u8, int B, int H, int W, void* pixels_f16, uint8_t* crop_u8,
                          void* patch_rows_f16, void* stream) {
  SafetyEngine* E = reinterpret_cast<SafetyEngine*>(e);
  if (int rc = frames_ok(E, frames_u8, B, H, W)) return rc;
  SDW_REQUIRE(B <= E->cfg.max_batch, "preprocess: B exceeds max_batch");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = E->prepare(H, W)) return rc;
  if (int rc = E->preprocess(frames_u8, B, H, W, static_cast<__half*>(pixels_f16), st, static_cast<__half*>(patch_rows_f16)))
    return rc;
  if (crop_u8)
    SDW_CUDA_OK(cudaMemcpyAsync(crop_u8, E->crop, static_cast<size_t>(B) * SAFETY_CROP * SAFETY_CROP * 3,
                                cudaMemcpyDeviceToDevice, st));
  return 0;
}

int sdw_safety_embed(sdw_safety* e, const uint8_t* frames_u8, int B, int H, int W, float* embeds_f32, int use_graph,
                     void* stream) {
  SafetyEngine* E = reinterpret_cast<SafetyEngine*>(e);
  if (int rc = frames_ok(E, frames_u8, B, H, W)) return rc;
  SDW_REQUIRE(embeds_f32, "null embeddings");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDW_REQUIRE(!use_graph || st != nullptr, "graph capture needs a real stream, not the legacy default stream 0");
  return E->run(frames_u8, nullptr, B, H, W, nullptr, nullptr, embeds_f32, use_graph, st);
}

int sdw_safety_scores(const float* embeds_f32, int B, int D, const float* special, const float* special_w, int ns,
                      const float* concepts, const float* concept_w, int nc, int32_t* flags, float* cos_f32,
                      double* scores_f64, uint8_t* frames_u8, int64_t frame_bytes, void* stream) {
  SDW_REQUIRE(embeds_f32 && flags && (ns == 0 || (special && special_w)) && (nc == 0 || (concepts && concept_w)), "null");
  SDW_REQUIRE(B >= 1 && B <= 65535 && D >= 1, "scores: bad B / D");
  SDW_REQUIRE(ns >= 0 && nc >= 0 && ns + nc >= 1 && ns + nc <= SAFETY_MAX_SCORES, "scores: 1..64 concepts in all");
  SDW_REQUIRE(!frames_u8 || frame_bytes >= 0, "scores: frame_bytes");
  safety_score_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(embeds_f32, D, special, special_w, ns, concepts,
                                                                          concept_w, nc, flags, cos_f32, scores_f64,
                                                                          frames_u8, frame_bytes);
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

// tooling: CUDA-event time of every op of one check of B frames of H x W (B <= max_batch), written as TSV lines
int sdw_safety_debug_profile(sdw_safety* e, const uint8_t* frames_u8, int B, int H, int W, const char* path, void* stream) {
  SafetyEngine* E = reinterpret_cast<SafetyEngine*>(e);
  if (int rc = frames_ok(E, frames_u8, B, H, W)) return rc;
  SDW_REQUIRE(path && B <= E->cfg.max_batch, "profile: path, B <= max_batch");
  if (int rc = E->prepare(H, W)) return rc;
  SafetyTower* t = E->tower(B);
  if (!t) return 1;
  OpList ops;
  ops.add("preprocess (resize, crop, normalise, patch rows)",
          [=](cudaStream_t st, int) { return E->preprocess(frames_u8, B, H, W, nullptr, st); });
  ops.append(t->ops);
  int32_t* flags = reinterpret_cast<int32_t*>(E->pooled32);  // dead after the projection
  ops.add("concept scores",
          [=](cudaStream_t st, int) { return E->scores(E->embeds, B, flags, nullptr, nullptr, nullptr, 0, st); });
  FILE* f = std::fopen(path, "w");
  SDW_REQUIRE(f, "cannot open the profile file");
  int rc = profile_ops(f, "safety", ops, static_cast<cudaStream_t>(stream), 0);
  std::fclose(f);
  if (rc) return rc;
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
