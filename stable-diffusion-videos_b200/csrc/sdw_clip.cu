// sdw_clip.cu — the CLIP text tower behind `embed_text` (stable_diffusion_pipeline.py:809-820) and the per-call ""
// encode (P:341-348), natively: token + position embedding, N pre-LN transformer layers with a causal mask, final
// LayerNorm; the caller takes last_hidden_state [B][77][hidden] (P:306, 819).
//
// SD-1.x: ViT-L/14 text tower (12 layers, 768 wide, 12 heads x 64, MLP 3072, quick-GELU); SD-2.x: OpenCLIP-H (23 used
// layers, 1024 wide, 16 heads x 64, MLP 4096, GELU) — both are configurations of this engine.  The linears run on the
// wgmma GEMM of sdw_gemm.cu (M = 77 B rows: one or two 128-row tiles), LayerNorm on sdw_norm.cu's kernel; the
// 77 x 77 causal attention per head and the embedding gather are small CUDA-core kernels here (13 GFLOP per prompt: the
// tower is a feed of the hot loop, not part of it).  State-dict names are transformers' `CLIPTextModel` keys.
// The encoder layers (`ClipEncoder`) also make the safety checker's image tower (sdw_safety.cu), there not causal.
#include "sdw_internal.h"
#include "sdw_ptx.cuh"

#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/sdwalk.h"

namespace sdw {

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
__global__ void clip_embed_kernel(const int32_t* __restrict__ ids, const __half* __restrict__ tok,
                                  const __half* __restrict__ pos, int P, int H, int vocab, __half* __restrict__ x) {
  const int row = blockIdx.x;  // b * P + p
  int id = ids[row];
  id = min(max(id, 0), vocab - 1);
  const __half2* t2 = reinterpret_cast<const __half2*>(tok + static_cast<int64_t>(id) * H);
  const __half2* p2 = reinterpret_cast<const __half2*>(pos + static_cast<int64_t>(row % P) * H);
  __half2* o2 = reinterpret_cast<__half2*>(x + static_cast<int64_t>(row) * H);
  for (int i = threadIdx.x; i < H / 2; i += blockDim.x) {
    const float2 a = __half22float2(t2[i]), b = __half22float2(p2[i]);
    o2[i] = __floats2half2_rn(a.x + b.x, a.y + b.y);
  }
}

// causal self-attention of one (head, sample): qkv [T][3H] (q | k | v column blocks, head h at columns h*64), out [T][H].
// 128 threads; K and V of the head staged in shared memory; warp w owns query rows w, w+4, ...
template <int MAXP>
__global__ void __launch_bounds__(128) clip_attn_kernel(const __half* __restrict__ qkv, int P, int H,
                                                        __half* __restrict__ out) {
  constexpr int D = 64;
  __shared__ __half ks[MAXP][D + 2];  // fp16 as stored; +2 keeps the per-lane rows on different banks
  __shared__ __half vs[MAXP][D];
  __shared__ float qs[4][D];
  const int head = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* base = qkv + static_cast<int64_t>(b) * P * 3 * H + head * D;
  for (int i = threadIdx.x; i < P * D; i += blockDim.x) {
    const int r = i / D, c = i % D;
    ks[r][c] = base[static_cast<int64_t>(r) * 3 * H + H + c];
    vs[r][c] = base[static_cast<int64_t>(r) * 3 * H + 2 * H + c];
  }
  __syncthreads();
  const float scale = 0.125f;  // 64^-1/2
  for (int i = warp; i < P; i += 4) {
    qs[warp][lane] = __half2float(base[static_cast<int64_t>(i) * 3 * H + lane]) * scale;
    qs[warp][lane + 32] = __half2float(base[static_cast<int64_t>(i) * 3 * H + lane + 32]) * scale;
    __syncwarp();
    float s[(MAXP + 31) / 32];
    float m = -INFINITY;
#pragma unroll
    for (int t = 0; t < (MAXP + 31) / 32; ++t) {
      const int j = t * 32 + lane;
      float acc = -INFINITY;
      if (j <= i) {  // causal mask: key j is visible to query i iff j <= i
        acc = 0.f;
#pragma unroll 16
        for (int c = 0; c < D; ++c) acc = fmaf(qs[warp][c], __half2float(ks[j][c]), acc);
      }
      s[t] = acc;
      m = fmaxf(m, acc);
    }
    m = warp_max(m);
    float l = 0.f;
#pragma unroll
    for (int t = 0; t < (MAXP + 31) / 32; ++t) {
      s[t] = (t * 32 + lane <= i) ? __expf(s[t] - m) : 0.f;
      l += s[t];
    }
    l = warp_sum(l);
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j <= i; ++j) {
      const float pj = __shfl_sync(0xffffffffu, s[j >> 5], j & 31);
      o0 = fmaf(pj, __half2float(vs[j][lane]), o0);
      o1 = fmaf(pj, __half2float(vs[j][lane + 32]), o1);
    }
    const float inv = 1.f / l;
    __half* orow = out + (static_cast<int64_t>(b) * P + i) * H + head * D;
    orow[lane] = __float2half_rn(o0 * inv);
    orow[lane + 32] = __float2half_rn(o1 * inv);
    __syncwarp();
  }
}

__global__ void clip_act_kernel(__half* __restrict__ x, int64_t n, int gelu_erf) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = __half2float(x[i]);
  // erf GELU as 0.5 v erfc(-v / sqrt 2): 1 + erf(x) cancels for x < -2 and loses up to 2 fp16 ulps of the result
  const float y = gelu_erf ? 0.5f * v * erfcf(v * -0.70710678118654752f) : v / (1.f + __expf(-1.702f * v));
  x[i] = __float2half_rn(y);
}

static int clip_attention(const __half* qkv, int B, int P, int heads, __half* out, cudaStream_t st) {
  clip_attn_kernel<96><<<dim3(heads, B), 128, 0, st>>>(qkv, P, heads * 64, out);
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

static int clip_act(__half* x, int64_t n, int gelu_erf, cudaStream_t st) {
  clip_act_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(x, n, gelu_erf);
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// the encoder
// ---------------------------------------------------------------------------------------------
void ClipEncoder::layout(Arena& arena, ParamTable& params, const std::string& prefix, int n_layers, int H, int I) {
  hidden = H;
  intermediate = I;
  layers.assign(n_layers, Layer{});
  for (int i = 0; i < n_layers; ++i) {
    Layer& L = layers[i];
    const std::string p = prefix + std::to_string(i) + ".";
    L.ln1_g = arena.take<float>(H); L.ln1_b = arena.take<float>(H);
    L.ln2_g = arena.take<float>(H); L.ln2_b = arena.take<float>(H);
    L.bqkv = arena.take<float>(3 * H); L.bo = arena.take<float>(H);
    L.b1 = arena.take<float>(I); L.b2 = arena.take<float>(H);
    L.wqkv = arena.take<__half>(static_cast<size_t>(3) * H * H);
    L.wo = arena.take<__half>(static_cast<size_t>(H) * H);
    L.w1 = arena.take<__half>(static_cast<size_t>(I) * H);
    L.w2 = arena.take<__half>(static_cast<size_t>(H) * I);
    params.add(p + "layer_norm1.weight", VEC, L.ln1_g, H); params.add(p + "layer_norm1.bias", VEC, L.ln1_b, H);
    params.add(p + "layer_norm2.weight", VEC, L.ln2_g, H); params.add(p + "layer_norm2.bias", VEC, L.ln2_b, H);
    const char* qkvn[3] = {"q_proj", "k_proj", "v_proj"};
    for (int k = 0; k < 3; ++k) {
      params.add(p + "self_attn." + qkvn[k] + ".weight", PACKED, L.wqkv ? L.wqkv + static_cast<size_t>(k) * H * H : nullptr,
                 static_cast<int64_t>(H) * H, H, H);
      params.add(p + "self_attn." + qkvn[k] + ".bias", VEC, L.bqkv ? L.bqkv + k * H : nullptr, H);
    }
    params.add(p + "self_attn.out_proj.weight", PACKED, L.wo, static_cast<int64_t>(H) * H, H, H);
    params.add(p + "self_attn.out_proj.bias", VEC, L.bo, H);
    params.add(p + "mlp.fc1.weight", PACKED, L.w1, static_cast<int64_t>(I) * H, I, H);
    params.add(p + "mlp.fc1.bias", VEC, L.b1, I);
    params.add(p + "mlp.fc2.weight", PACKED, L.w2, static_cast<int64_t>(H) * I, H, I);
    params.add(p + "mlp.fc2.bias", VEC, L.b2, H);
  }
}

// out[T][N] = a[T][K] w^T + bias (+ resid)
static GemmDesc linear_desc(const __half* a, int64_t T, int K, const __half* w, int N, const float* bias,
                            const __half* resid, __half* out) {
  GemmDesc d;
  d.A = a; d.C = K; d.W = static_cast<int>(T); d.H = 1; d.B = 1; d.sW = K;
  d.Wt = w; d.N = N; d.bias = bias; d.resid = resid; d.out = out; d.ldc = N;
  return d;
}

int ClipEncoder::emit(OpList& ops, int B, int P, float eps, int gelu_erf, bool causal, const Buffers& b) const {
  const int H = hidden, I = intermediate, heads = H / 64;
  const int64_t T = static_cast<int64_t>(B) * P;
  __half *x = b.x, *y = b.y, *h = b.h, *ff = b.ff, *qkv = b.qkv;
  for (size_t i = 0; i < layers.size(); ++i) {
    const Layer& L = layers[i];
    const std::string p = "layer " + std::to_string(i) + " ";
    ops.add(p + "ln1", [=](cudaStream_t st, int) { return layernorm(x, H, T, H, L.ln1_g, L.ln1_b, eps, h, H, st); });
    GemmDesc g = linear_desc(h, T, H, L.wqkv, 3 * H, L.bqkv, nullptr, qkv);
    if (causal) {
      if (int e = ops.add_gemm(g, p + "qkv")) return e;
      ops.add(p + "attention", [=](cudaStream_t st, int) { return clip_attention(qkv, B, P, heads, h, st); });
    } else {
      g.ldc = 2 * H;
      g.mode = GEMM_QKV_VT;
      g.vt_col0 = 2 * H; g.vt_d = 64; g.vt_heads = heads; g.vt_ntok = P; g.vt = b.vt; g.vt_ld = b.vt_ld;
      if (int e = ops.add_gemm(g, p + "qkv + V^T")) return e;
      AttnDesc ad;
      ad.q = qkv; ad.q_ld = 2 * H; ad.k = qkv + H; ad.k_ld = 2 * H; ad.vt = b.vt; ad.vt_ld = b.vt_ld;
      ad.B = B; ad.Nq = P; ad.Nk = P; ad.heads = heads; ad.d = 64;
      ad.out = h; ad.out_ld = H;
      auto AL = std::make_shared<AttnLaunch>();
      if (int e = plan_attention(ad, AL.get())) return e;
      ops.add(p + "attention", [AL](cudaStream_t st, int) { return launch_attention(*AL, st); });
    }
    if (int e = ops.add_gemm(linear_desc(h, T, H, L.wo, H, L.bo, x, y), p + "out_proj + x")) return e;
    std::swap(x, y);
    ops.add(p + "ln2", [=](cudaStream_t st, int) { return layernorm(x, H, T, H, L.ln2_g, L.ln2_b, eps, h, H, st); });
    if (int e = ops.add_gemm(linear_desc(h, T, H, L.w1, I, L.b1, nullptr, ff), p + "fc1")) return e;
    ops.add(p + "act", [=](cudaStream_t st, int) { return clip_act(ff, T * I, gelu_erf, st); });
    if (int e = ops.add_gemm(linear_desc(ff, T, I, L.w2, H, L.b2, x, y), p + "fc2 + x")) return e;
    std::swap(x, y);
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// engine
// ---------------------------------------------------------------------------------------------
struct ClipEngine {
  sdw_clip_config cfg;
  Arena arena{256};
  size_t cap = 0;
  ParamTable params;
  ClipEncoder enc;
  __half *tok = nullptr, *pos = nullptr;
  float *lnf_g = nullptr, *lnf_b = nullptr;
  __half *x0 = nullptr, *x1 = nullptr, *h = nullptr, *qkv = nullptr, *ff = nullptr;
  std::map<int, OpList> towers;  // encoder ops per batch size

  void layout(void* base) {
    const sdw_clip_config& c = cfg;
    const int H = c.hidden, I = c.intermediate;
    arena.reset(base);
    params.clear(base != nullptr);
    towers.clear();
    tok = arena.take<__half>(static_cast<size_t>(c.vocab) * H);
    pos = arena.take<__half>(static_cast<size_t>(c.max_positions) * H);
    params.add("text_model.embeddings.token_embedding.weight", RAW, tok, static_cast<int64_t>(c.vocab) * H);
    params.add("text_model.embeddings.position_embedding.weight", RAW, pos, static_cast<int64_t>(c.max_positions) * H);
    enc.layout(arena, params, "text_model.encoder.layers.", c.layers, H, I);
    lnf_g = arena.take<float>(H); lnf_b = arena.take<float>(H);
    params.add("text_model.final_layer_norm.weight", VEC, lnf_g, H);
    params.add("text_model.final_layer_norm.bias", VEC, lnf_b, H);
    const size_t T = static_cast<size_t>(c.max_batch) * c.max_positions;
    x0 = arena.take<__half>(T * H); x1 = arena.take<__half>(T * H); h = arena.take<__half>(T * H);
    qkv = arena.take<__half>(T * 3 * H); ff = arena.take<__half>(T * I);
  }

  // the encoder of B prompts, from the embeddings in x0 to its result in x0; planned on first use
  const OpList* tower(int B) {
    auto it = towers.find(B);
    if (it != towers.end()) return &it->second;
    OpList ops;
    ClipEncoder::Buffers b;
    b.x = x0; b.y = x1; b.h = h; b.ff = ff; b.qkv = qkv;
    if (enc.emit(ops, B, cfg.max_positions, cfg.eps, cfg.act_gelu_erf, true, b)) return nullptr;
    return &(towers[B] = std::move(ops));
  }
};

}  // namespace sdw

using namespace sdw;

extern "C" {

int sdw_clip_create(const sdw_clip_config* cfg, sdw_clip** out) {
  SDW_REQUIRE(cfg && out, "null");
  SDW_REQUIRE(cfg->hidden % 64 == 0 && cfg->hidden == cfg->heads * 64, "CLIP text towers here have 64-wide heads");
  SDW_REQUIRE(cfg->intermediate % 64 == 0 && cfg->layers >= 1 && cfg->vocab >= 1, "bad CLIP configuration");
  SDW_REQUIRE(cfg->max_positions >= 1 && cfg->max_positions <= 96, "at most 96 positions (77 in every SD checkpoint)");
  SDW_REQUIRE(cfg->max_batch >= 1, "max_batch");
  ClipEngine* E = new ClipEngine();
  E->cfg = *cfg;
  E->layout(nullptr);
  E->cap = E->arena.off;
  *out = reinterpret_cast<sdw_clip*>(E);
  return 0;
}

void sdw_clip_destroy(sdw_clip* e) { delete reinterpret_cast<ClipEngine*>(e); }

int sdw_clip_arena_bytes(const sdw_clip* e, uint64_t* bytes) {
  const ClipEngine* E = reinterpret_cast<const ClipEngine*>(e);
  SDW_REQUIRE(E && bytes, "null");
  *bytes = E->cap + 256;
  return 0;
}

int sdw_clip_bind(sdw_clip* e, void* arena, uint64_t bytes) {
  ClipEngine* E = reinterpret_cast<ClipEngine*>(e);
  SDW_REQUIRE(E && arena, "null");
  SDW_REQUIRE(bytes >= E->cap + 256, "arena too small");
  SDW_REQUIRE((reinterpret_cast<uintptr_t>(arena) & 255) == 0, "arena must be 256-byte aligned");
  E->layout(arena);
  return 0;
}

int sdw_clip_num_params(const sdw_clip* e) { return e ? reinterpret_cast<const ClipEngine*>(e)->params.size() : 0; }

int sdw_clip_param_info(const sdw_clip* e, int index, const char** name, int64_t* numel) {
  SDW_REQUIRE(e, "null");
  return reinterpret_cast<const ClipEngine*>(e)->params.info(index, name, numel);
}

int sdw_clip_load_param(sdw_clip* e, const char* name, const void* data_f16, int64_t numel, void* stream) {
  SDW_REQUIRE(e, "null");
  return reinterpret_cast<ClipEngine*>(e)->params.load(name, data_f16, numel, static_cast<cudaStream_t>(stream));
}

int sdw_clip_missing_params(const sdw_clip* e, const char** first_missing) {
  return e ? reinterpret_cast<const ClipEngine*>(e)->params.missing(first_missing) : -1;
}

int sdw_clip_forward(sdw_clip* e, const int32_t* ids, int B, void* out_f16, void* stream) {
  ClipEngine* E = reinterpret_cast<ClipEngine*>(e);
  SDW_REQUIRE(E && ids && out_f16 && E->params.bound, "null / engine not bound");
  const sdw_clip_config& c = E->cfg;
  SDW_REQUIRE(B >= 1 && B <= c.max_batch, "batch exceeds max_batch");
  SDW_REQUIRE(E->params.missing(nullptr) == 0, "CLIP parameters not loaded");
  const OpList* t = E->tower(B);
  if (!t) return 1;
  // no CUDA graph: the caller's stream may be the legacy default stream, which cannot be captured
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int P = c.max_positions, H = c.hidden;
  const int64_t T = static_cast<int64_t>(B) * P;
  clip_embed_kernel<<<static_cast<unsigned>(T), 128, 0, st>>>(ids, E->tok, E->pos, P, H, c.vocab, E->x0);
  SDW_CUDA_OK(cudaGetLastError());
  if (int rc = t->run(st, 0)) return rc;
  return layernorm(E->x0, H, T, H, E->lnf_g, E->lnf_b, c.eps, static_cast<__half*>(out_f16), H, st);
}

// the tower's three kernels on their own (tests / tooling)
int sdw_clip_embed(const int32_t* ids, const void* tok, const void* pos, int rows, int P, int H, int vocab, void* x,
                   void* stream) {
  SDW_REQUIRE(ids && tok && pos && x, "null");
  SDW_REQUIRE(rows >= 1 && P >= 1 && vocab >= 1 && H >= 8 && H % 8 == 0, "CLIP embedding: rows, P, vocab >= 1, H % 8 == 0");
  SDW_REQUIRE(((reinterpret_cast<uintptr_t>(tok) | reinterpret_cast<uintptr_t>(pos) | reinterpret_cast<uintptr_t>(x)) & 3) == 0,
              "CLIP embedding: tok, pos and x must be 4-byte aligned");
  clip_embed_kernel<<<static_cast<unsigned>(rows), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      ids, static_cast<const __half*>(tok), static_cast<const __half*>(pos), P, H, vocab, static_cast<__half*>(x));
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

int sdw_clip_attention(const void* qkv, int B, int P, int heads, void* out, void* stream) {
  SDW_REQUIRE(qkv && out, "null");
  SDW_REQUIRE(P >= 1 && P <= 96, "CLIP attention: 1 <= P <= 96 (the kernel stages K and V of 96 positions)");
  SDW_REQUIRE(B >= 1 && B <= 65535 && heads >= 1 && heads <= 65535, "CLIP attention: bad B / heads");
  return clip_attention(static_cast<const __half*>(qkv), B, P, heads, static_cast<__half*>(out),
                        static_cast<cudaStream_t>(stream));
}

int sdw_clip_act(void* x, int64_t n, int gelu_erf, void* stream) {
  SDW_REQUIRE(x && n >= 0 && (gelu_erf == 0 || gelu_erf == 1), "CLIP activation: null x, n < 0 or bad activation");
  SDW_REQUIRE(n <= int64_t(1) << 38, "CLIP activation: n too large for one launch");
  if (n == 0) return 0;
  return clip_act(static_cast<__half*>(x), n, gelu_erf, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
