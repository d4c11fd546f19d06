// sdw_attn.cu — fused (flash) attention on wgmma for the UNet's self- and cross-attention
// (the SDPA inside `BasicTransformerBlock`, reached from stable_diffusion_pipeline.py:418).
//
//   O[b, q, h*d:(h+1)*d] = softmax(Q_h K_h^T * d^-1/2) V_h          per (batch b, head h), fp16 in / fp16 out
//
// Nothing but Q, K, V^T tiles and the O tile touches HBM.  One CTA = one 128-query tile of one (b, h):
//   warp 8    : TMA producer — the Q tile once, then K and V^T tiles of BKV keys into a ring of ST stages.  The head
//               dimension is loaded in 64-column boxes whose columns beyond d are zero-filled by TMA, and V^T rows
//               beyond d likewise, so padding needs no code.
//   warps 0-7 : two consumer warpgroups, 64 query rows each.  Per KV tile: S = Q K^T (wgmma m64nBKVk16, operands in
//               shared memory, fp32 scores in registers), online softmax in registers (a query row lives in the four
//               lanes of a quad), P rounded to fp16 and fed straight from registers as the A operand of
//               O += P V (wgmma m64nDVPk16, register-A form), then the stage is released.  The two warpgroups
//               interleave on the SM: one's exponentials overlap the other's MMAs.
// Ordering is carried by mbarriers only.
#include "sdw_internal.h"
#include "sdw_ptx.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace sdw {

static constexpr int ATT_THREADS = 288;  // two consumer warpgroups + one producer warp
static constexpr int ATT_BQ = 128;
static constexpr int ATT_ST = 3;

struct alignas(64) AttnKParams {
  CUtensorMap mapQ, mapK, mapV;
  int Nq, Nk, d, heads;
  int dk_steps;          // ceil(d / 16)
  float scale_log2e;     // d^-1/2 * log2(e)
  __half* out;
  int64_t out_ld;
  int vec2;              // 1: output rows allow 4-byte column-pair stores
};

// DKC 64-column chunks of the head dimension for Q and K; DVP = head dimension padded for the PV tile width
template <int DKC, int DVP, int BKV>
struct AttnCfg {
  static constexpr int Q_BYTES = DKC * ATT_BQ * 128;
  static constexpr int K_CHUNK = BKV * 128;
  static constexpr int K_STAGE = DKC * K_CHUNK;
  static constexpr int V_BOX = DVP * 128;  // one 64-key box of V^T rows
  static constexpr int V_STAGE = (BKV / 64) * V_BOX;
  static constexpr int SMEM = 1024 /*align*/ + 1024 /*barriers*/ + Q_BYTES + ATT_ST * (K_STAGE + V_STAGE);
  static_assert(V_BOX % 1024 == 0 && K_CHUNK % 1024 == 0, "swizzle atoms must stay 1024-byte aligned");
  static_assert(SMEM <= 227 * 1024, "shared memory");
};

template <int DKC, int DVP, int BKV>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_kernel(const __grid_constant__ AttnKParams p) {
  using Cfg = AttnCfg<DKC, DVP, BKV>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* full_bar = q_full + 1;
  uint64_t* empty_bar = full_bar + ATT_ST;
  uint8_t* sQ = smem + 1024;
  uint8_t* sK = sQ + Cfg::Q_BYTES;
  uint8_t* sV = sK + ATT_ST * Cfg::K_STAGE;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nkv = (p.Nk + BKV - 1) / BKV;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&p.mapQ);
    tma_prefetch_desc(&p.mapK);
    tma_prefetch_desc(&p.mapV);
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_ST; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp == 8) {
    // =========================== TMA producer ===============================
    if (lane == 0) {
      mbar_expect_tx(q_full, Cfg::Q_BYTES);
#pragma unroll
      for (int c = 0; c < DKC; ++c) tma_load_4d(&p.mapQ, q_full, sQ + c * ATT_BQ * 128, 64 * c, qt * ATT_BQ, h, b);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], Cfg::K_STAGE + Cfg::V_STAGE);
#pragma unroll
        for (int c = 0; c < DKC; ++c)
          tma_load_4d(&p.mapK, &full_bar[stage], sK + stage * Cfg::K_STAGE + c * Cfg::K_CHUNK, 64 * c, j * BKV, h, b);
#pragma unroll
        for (int i = 0; i < BKV / 64; ++i)
          tma_load_4d(&p.mapV, &full_bar[stage], sV + stage * Cfg::V_STAGE + i * Cfg::V_BOX, j * BKV + 64 * i, 0, h, b);
        if (++stage == ATT_ST) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // =========================== consumers ======================================
  const int wg = warp >> 2;
  const int q2 = 2 * (lane & 3);
  float o[DVP / 2];
#pragma unroll
  for (int i = 0; i < DVP / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t q_base = smem_u32(sQ) + wg * (64 * 128);
  mbar_wait(q_full, 0);

  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < nkv; ++j) {
    mbar_wait(&full_bar[stage], phase);
    // ---- S = Q K^T ----
    float s[BKV / 2];
    wgmma_fence();
    const uint32_t k_base = smem_u32(sK + stage * Cfg::K_STAGE);
#pragma unroll
    for (int c = 0; c < DKC; ++c) {
      const uint64_t dq = make_desc_k_sw128(q_base + c * ATT_BQ * 128);
      const uint64_t dk = make_desc_k_sw128(k_base + c * Cfg::K_CHUNK);
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int kk = 4 * c + ks;
        if (kk < p.dk_steps) Wgmma<BKV>::ss(s, dq + 2 * ks, dk + 2 * ks, kk > 0 ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // ---- online softmax (base 2), keys beyond Nk masked ----
    const int valid = p.Nk - j * BKV;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jb = 0; jb < BKV / 8; ++jb)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& x = s[4 * jb + 2 * hh + e];
          x = (8 * jb + q2 + e < valid) ? x * p.scale_log2e : -INFINITY;
          mx[hh] = fmaxf(mx[hh], x);
        }
    float corr[2], sum[2] = {0.f, 0.f};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      const float mn = fmaxf(m[hh], mx[hh]);
      corr[hh] = ex2f(m[hh] - mn);
      m[hh] = mn;
    }
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int jb = 0; jb < BKV / 8; ++jb) {
      float e0 = ex2f(s[4 * jb + 0] - m[0]), e1 = ex2f(s[4 * jb + 1] - m[0]);
      float e2 = ex2f(s[4 * jb + 2] - m[1]), e3 = ex2f(s[4 * jb + 3] - m[1]);
      sum[0] += e0 + e1;
      sum[1] += e2 + e3;
      // A fragment of k16 block jb / 2: {row r, k 2q..}, {row r+8, k 2q..}, {row r, k 8+2q..}, {row r+8, k 8+2q..}
      pa[jb / 2][2 * (jb & 1) + 0] = pack_h2(e0, e1);
      pa[jb / 2][2 * (jb & 1) + 1] = pack_h2(e2, e3);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) l[hh] = l[hh] * corr[hh] + sum[hh];
#pragma unroll
    for (int jb = 0; jb < DVP / 8; ++jb) {
      o[4 * jb + 0] *= corr[0];
      o[4 * jb + 1] *= corr[0];
      o[4 * jb + 2] *= corr[1];
      o[4 * jb + 3] *= corr[1];
    }

    // ---- O += P V ----
    wgmma_fence();
    const uint32_t v_base = smem_u32(sV + stage * Cfg::V_STAGE);
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      const uint64_t dv = make_desc_k_sw128(v_base + (kk / 4) * Cfg::V_BOX);
      Wgmma<DVP>::rs(o, pa[kk], dv + 2 * (kk % 4), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == ATT_ST) {
      stage = 0;
      phase ^= 1;
    }
  }

  // ---- normalise and store ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    const int q = qt * ATT_BQ + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * hh;
    if (q >= p.Nq) continue;
    const float inv = 1.f / l[hh];
    __half* dst = p.out + (static_cast<int64_t>(b) * p.Nq + q) * p.out_ld + static_cast<int64_t>(h) * p.d;
#pragma unroll
    for (int jb = 0; jb < DVP / 8; ++jb) {
      const int col = 8 * jb + q2;
      if (col >= p.d) continue;  // d % 8 == 0: col + 1 < d too
      const float v0 = o[4 * jb + 2 * hh] * inv, v1 = o[4 * jb + 2 * hh + 1] * inv;
      if (p.vec2) {
        *reinterpret_cast<uint32_t*>(dst + col) = pack_h2(v0, v1);
      } else {
        dst[col] = __float2half_rn(v0);
        dst[col + 1] = __float2half_rn(v1);
      }
    }
  }
}

// =============================================================================================
// host
// =============================================================================================
// variants: 0..3 head dim <= 16 / 32 / 48 / 64 (BKV 128, one 64-column head-dim chunk)
//           4    head dim <= 80  (BKV 64, two chunks)
//           5    head dim <= 160 (BKV 64, three chunks)
struct AttnLaunchImpl {
  AttnKParams p;
  dim3 grid;
  int variant;
};

template <int DKC, int DVP, int BKV>
static cudaError_t launch_fwd(const AttnLaunchImpl* I, cudaStream_t stream) {
  using Cfg = AttnCfg<DKC, DVP, BKV>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_kernel<DKC, DVP, BKV>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  return launch_pdl(attn_kernel<DKC, DVP, BKV>, I->grid, dim3(ATT_THREADS), Cfg::SMEM, stream, I->p);
}

bool attn_supported(int d) { return d % 8 == 0 && d >= 8 && d <= 160; }

static int variant_for(int d) {
  if (d <= 64) return d <= 16 ? 0 : (d <= 32 ? 1 : (d <= 48 ? 2 : 3));
  return d <= 80 ? 4 : 5;
}

int plan_attention(const AttnDesc& a, AttnLaunch* L) {
  SDW_REQUIRE(attn_supported(a.d), "flash attention supports head dims 8..160 (multiples of 8)");
  SDW_REQUIRE(a.q && a.k && a.vt && a.out, "null operand");
  SDW_REQUIRE(a.Nq > 0 && a.Nk > 0 && a.heads > 0 && a.B > 0, "empty attention");
  SDW_REQUIRE(a.heads <= 65535 && a.B <= 65535, "attention grid too large");
  static_assert(sizeof(AttnLaunchImpl) <= sizeof(AttnLaunch::storage), "AttnLaunch storage too small");
  AttnLaunchImpl* I = reinterpret_cast<AttnLaunchImpl*>(L->storage);
  std::memset(I, 0, sizeof(*I));
  I->variant = variant_for(a.d);
  const int bkv = I->variant >= 4 ? 64 : 128;
  const int dvp_tab[6] = {16, 32, 48, 64, 80, 160};
  const int dvp = dvp_tab[I->variant];
  AttnKParams& p = I->p;
  p.Nq = a.Nq; p.Nk = a.Nk; p.d = a.d; p.heads = a.heads;
  p.dk_steps = (a.d + 15) / 16;
  p.scale_log2e = (1.f / std::sqrt(static_cast<float>(a.d))) * 1.4426950408889634f;
  p.out = a.out; p.out_ld = a.out_ld;
  p.vec2 = (a.out_ld % 2 == 0) && (reinterpret_cast<uintptr_t>(a.out) & 3) == 0;
  const int qtiles = (a.Nq + ATT_BQ - 1) / ATT_BQ;
  I->grid = dim3(qtiles, a.heads, a.B);
  {
    uint64_t dims[4] = {static_cast<uint64_t>(a.d), static_cast<uint64_t>(a.Nq), static_cast<uint64_t>(a.heads),
                        static_cast<uint64_t>(a.B)};
    uint64_t str[4] = {1, static_cast<uint64_t>(a.q_ld), static_cast<uint64_t>(a.d),
                       static_cast<uint64_t>(a.Nq) * a.q_ld};
    uint32_t box[4] = {64, ATT_BQ, 1, 1};
    if (int e = encode_map(&p.mapQ, a.q, 4, dims, str, box)) return e;
  }
  {
    uint64_t dims[4] = {static_cast<uint64_t>(a.d), static_cast<uint64_t>(a.Nk), static_cast<uint64_t>(a.heads),
                        static_cast<uint64_t>(a.B)};
    uint64_t str[4] = {1, static_cast<uint64_t>(a.k_ld), static_cast<uint64_t>(a.d),
                       static_cast<uint64_t>(a.Nk) * a.k_ld};
    uint32_t box[4] = {64, static_cast<uint32_t>(bkv), 1, 1};
    if (int e = encode_map(&p.mapK, a.k, 4, dims, str, box)) return e;
  }
  {
    uint64_t dims[4] = {static_cast<uint64_t>(a.Nk), static_cast<uint64_t>(a.d), static_cast<uint64_t>(a.heads),
                        static_cast<uint64_t>(a.B)};
    uint64_t str[4] = {1, static_cast<uint64_t>(a.vt_ld), static_cast<uint64_t>(a.d) * a.vt_ld,
                       static_cast<uint64_t>(a.heads) * a.d * a.vt_ld};
    uint32_t box[4] = {64, static_cast<uint32_t>(dvp), 1, 1};
    if (int e = encode_map(&p.mapV, a.vt, 4, dims, str, box)) return e;
  }
  return 0;
}

// planner introspection (host only): {variant, query tiles per CTA, grid.x, grid.y, grid.z}
void attention_plan_info(const AttnLaunch& L, int out[5]) {
  const AttnLaunchImpl* I = reinterpret_cast<const AttnLaunchImpl*>(L.storage);
  out[0] = I->variant;
  out[1] = 1;
  out[2] = static_cast<int>(I->grid.x);
  out[3] = static_cast<int>(I->grid.y);
  out[4] = static_cast<int>(I->grid.z);
}

int launch_attention(const AttnLaunch& L, cudaStream_t stream) {
  const AttnLaunchImpl* I = reinterpret_cast<const AttnLaunchImpl*>(L.storage);
  switch (I->variant) {
    case 0: SDW_CUDA_OK((launch_fwd<1, 16, 128>(I, stream))); break;
    case 1: SDW_CUDA_OK((launch_fwd<1, 32, 128>(I, stream))); break;
    case 2: SDW_CUDA_OK((launch_fwd<1, 48, 128>(I, stream))); break;
    case 3: SDW_CUDA_OK((launch_fwd<1, 64, 128>(I, stream))); break;
    case 4: SDW_CUDA_OK((launch_fwd<2, 80, 64>(I, stream))); break;
    case 5: SDW_CUDA_OK((launch_fwd<3, 160, 64>(I, stream))); break;
    default: set_error("bad attention variant"); return 1;
  }
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sdw
