// sdw_attn.cu — fused (flash) attention on wgmma for the UNet's self- and cross-attention
// (the SDPA inside `BasicTransformerBlock`, reached from stable_diffusion_pipeline.py:418).
//
//   O[b, q, h*d:(h+1)*d] = softmax(Q_h K_h^T * d^-1/2) V_h          per (batch b, head h), fp16 in / fp16 out
//
// Nothing but Q, K, V^T tiles and the O tile touches HBM.  One CTA = one 128-query tile of one (b, h), 384 threads:
//   warpgroup 2 (warps 8-11): producer, its registers handed to the consumers (setmaxnreg).  One thread TMA-loads the Q
//               tile once, then K and V^T tiles of BKV keys into a ring of ST stages.  The head dimension is loaded
//               in 64-column boxes whose columns beyond d are zero-filled by TMA, and V^T rows beyond d likewise, so
//               padding needs no code: the QK^T k-step count is DVP / 16 for every d of a variant.
//   warpgroups 0, 1: consumers, 64 query rows each.  S = Q K^T is wgmma m64nBKVk16 with both operands in shared
//               memory and fp32 scores in registers; the online softmax runs in registers (a query row lives in the
//               four lanes of a quad); P is rounded to fp16 and fed straight from registers as the A operand of
//               O += P V (wgmma m64nDVPk16, register-A form).
// Two overlaps keep MUFU (the exponentials) and the tensor cores busy at the same time:
//   - within a warpgroup, KV tile j's scores are issued together with tile j-1's PV product, and the softmax of tile j
//     runs while that PV product is still in flight (wgmma_wait<1>); O is rescaled only after it has landed;
//   - between the warpgroups (ping-pong), named barriers order the MMA issues: a warpgroup issues its two GEMMs only
//     after the other has issued its own, so one warpgroup's exponentials run under the other's MMAs.  Every
//     warpgroup passes every barrier whatever its rows, and the order does not change any arithmetic: the result is
//     the same bits on every run.
// No accumulator register is written between a wgmma issue and its wait (the C7515 serialisation of ptxas).  Stage
// ordering is carried by mbarriers; a stage is released once the PV product that reads its V^T has completed.
#include "sdw_internal.h"
#include "sdw_ptx.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace sdw {

static constexpr int ATT_THREADS = 384;  // two consumer warpgroups + one producer warpgroup
static constexpr int ATT_BQ = 128;
static constexpr int ATT_ST = 4;
// launched at <= 168 registers per thread (64K / 384); the producer gives 128 x 144 of them to the consumers
static constexpr int ATT_PRODUCER_REGS = 24;
static constexpr int ATT_CONSUMER_REGS = 240;
static constexpr int ATT_BAR_PINGPONG = 1;  // named barriers 1 and 2: "consumer warpgroup 0 / 1 may issue its MMAs"

struct alignas(64) AttnKParams {
  CUtensorMap mapQ, mapK, mapV;
  int Nq, Nk, d, heads;
  float scale_log2e;     // d^-1/2 * log2(e)
  __half* out;
  int64_t out_ld;
  int vec2;              // 1: output rows allow 4-byte column-pair stores
};

// DKC 64-column chunks of the head dimension for Q and K; DVP = head dimension padded for the PV tile width
template <int DKC, int DVP, int BKV>
struct AttnCfg {
  static constexpr int KSTEPS = DVP / 16;  // QK^T k-steps of 16 head-dim columns
  static constexpr int Q_BYTES = DKC * ATT_BQ * 128;
  static constexpr int K_CHUNK = BKV * 128;
  static constexpr int K_STAGE = DKC * K_CHUNK;
  static constexpr int V_BOX = DVP * 128;  // one 64-key box of V^T rows
  static constexpr int V_STAGE = (BKV / 64) * V_BOX;
  static constexpr int SMEM = 1024 /*align*/ + 1024 /*barriers*/ + Q_BYTES + ATT_ST * (K_STAGE + V_STAGE);
  static_assert(KSTEPS <= 4 * DKC, "k-steps beyond the loaded head-dim chunks");
  static_assert(V_BOX % 1024 == 0 && K_CHUNK % 1024 == 0, "swizzle atoms must stay 1024-byte aligned");
  static_assert(SMEM <= 227 * 1024, "shared memory");
};

// S = Q K^T of one KV stage for the warpgroup's 64 rows (one wgmma group)
template <int DKC, int DVP, int BKV>
__device__ __forceinline__ void attn_issue_s(float (&s)[BKV / 2], uint32_t q_base, uint32_t k_base) {
  using Cfg = AttnCfg<DKC, DVP, BKV>;
#pragma unroll
  for (int kk = 0; kk < Cfg::KSTEPS; ++kk) {
    const uint64_t dq = make_desc_k_sw128(q_base + (kk / 4) * ATT_BQ * 128);
    const uint64_t dk = make_desc_k_sw128(k_base + (kk / 4) * Cfg::K_CHUNK);
    Wgmma<BKV>::ss(s, dq + 2 * (kk % 4), dk + 2 * (kk % 4), kk > 0 ? 1u : 0u);
  }
  wgmma_commit();
}

// O += P V of one KV stage (one wgmma group); P as fp16 A fragments in registers
template <int DKC, int DVP, int BKV>
__device__ __forceinline__ void attn_issue_pv(float (&o)[DVP / 2], const uint32_t (&pa)[BKV / 16][4], uint32_t v_base) {
  using Cfg = AttnCfg<DKC, DVP, BKV>;
#pragma unroll
  for (int kk = 0; kk < BKV / 16; ++kk)
    Wgmma<DVP>::rs(o, pa[kk], make_desc_k_sw128(v_base + (kk / 4) * Cfg::V_BOX) + 2 * (kk % 4), 1u);
  wgmma_commit();
}

// One KV tile's online-softmax step on the warpgroup's fp32 scores (row r in s[4jb + 0..1], row r + 8 in
// s[4jb + 2..3], columns 8jb + 2(lane % 4) + {0, 1}).  The running max m is kept in raw score units, so each
// probability is one FFMA and one ex2: 2^(s c - m c) with c = d^-1/2 log2(e).  s is replaced in place by these
// probabilities, l is updated, and corr receives the factor O must be rescaled by.  MASK: keys at columns >= valid
// get probability 0; only the last KV tile can be ragged.
template <int BKV, bool MASK>
__device__ __forceinline__ void attn_softmax(float (&s)[BKV / 2], int valid, float c, float (&m)[2], float (&l)[2],
                                             float (&corr)[2]) {
  const int q2 = 2 * (threadIdx.x & 3);
  // four partial maxima and two partial sums per row: short dependency chains, so the one warp of each warpgroup on
  // a scheduler is not left waiting on FMNMX / FADD latency
  float mx4[2][4];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
#pragma unroll
    for (int i = 0; i < 4; ++i) mx4[hh][i] = m[hh];
#pragma unroll
  for (int jb = 0; jb < BKV / 8; ++jb)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& x = s[4 * jb + 2 * hh + e];
        if (MASK && 8 * jb + q2 + e >= valid) x = -INFINITY;
        mx4[hh][2 * (jb & 1) + e] = fmaxf(mx4[hh][2 * (jb & 1) + e], x);
      }
  float mx[2], mc[2], sum[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    mx[hh] = fmaxf(fmaxf(mx4[hh][0], mx4[hh][1]), fmaxf(mx4[hh][2], mx4[hh][3]));
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    corr[hh] = ex2f((m[hh] - mx[hh]) * c);  // the first tile: 2^-inf = 0 (every tile holds a key, so mx is finite)
    m[hh] = mx[hh];
    mc[hh] = mx[hh] * c;
  }
#pragma unroll
  for (int jb = 0; jb < BKV / 8; ++jb)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float* x = &s[4 * jb + 2 * hh];
      x[0] = ex2f(fmaf(x[0], c, -mc[hh]));
      x[1] = ex2f(fmaf(x[1], c, -mc[hh]));
      sum[hh][jb & 1] += x[0] + x[1];
    }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) l[hh] = l[hh] * corr[hh] + (sum[hh][0] + sum[hh][1]);
}

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

  if (warp >= 8) {
    // =========================== TMA producer ===============================
    setmaxnreg_dec<ATT_PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
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
  setmaxnreg_inc<ATT_CONSUMER_REGS>();
  const int wg = warp >> 2;
  const uint32_t bar_mine = ATT_BAR_PINGPONG + wg, bar_other = ATT_BAR_PINGPONG + (wg ^ 1);
  const float c = p.scale_log2e;
  const int last_valid = p.Nk - (nkv - 1) * BKV;  // keys in the last KV tile
  float o[DVP / 2];
#pragma unroll
  for (int i = 0; i < DVP / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, corr[2];
  float s[BKV / 2];          // scores of the newest KV tile, then its probabilities
  uint32_t pa[BKV / 16][4];  // probabilities of the previous KV tile as fp16 A fragments, read by its PV product
  const uint32_t q_base = smem_u32(sQ) + wg * (64 * 128);

  // A fragment of k16 block kb: {row r, k 2q..}, {row r+8, k 2q..}, {row r, k 8+2q..}, {row r+8, k 8+2q..}
  auto pack_p = [&]() {
#pragma unroll
    for (int jb = 0; jb < BKV / 8; ++jb) {
      pa[jb / 2][2 * (jb & 1) + 0] = pack_h2(s[4 * jb + 0], s[4 * jb + 1]);
      pa[jb / 2][2 * (jb & 1) + 1] = pack_h2(s[4 * jb + 2], s[4 * jb + 3]);
    }
#pragma unroll
    for (int kb = 0; kb < BKV / 16; ++kb)
#pragma unroll
      for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(pa[kb][i])::"memory");
  };
  auto softmax = [&](int j) {
    if (j == nkv - 1 && last_valid < BKV)
      attn_softmax<BKV, true>(s, last_valid, c, m, l, corr);
    else
      attn_softmax<BKV, false>(s, BKV, c, m, l, corr);
  };

  // warpgroup 0 issues first; afterwards each warpgroup waits for the other's issue before its own (bar_mine) and
  // lets the other go once its own GEMMs are issued (bar_other).  Per CTA both warpgroups issue nkv + 1 times.
  if (wg == 1) named_bar_arrive(ATT_BAR_PINGPONG, 256);
  mbar_wait(q_full, 0);

  // ---- prologue: S of KV tile 0 ----
  mbar_wait(&full_bar[0], 0);
  named_bar_sync(bar_mine, 256);
  wgmma_fence();
  attn_issue_s<DKC, DVP, BKV>(s, q_base, smem_u32(sK));
  named_bar_arrive(bar_other, 256);
  wgmma_wait<0>();
  reg_fence(s);
  softmax(0);
  pack_p();

  int stage = 0;  // stage of KV tile j - 1
  uint32_t phase = 0;
  for (int j = 1; j < nkv; ++j) {
    const int next = stage + 1 == ATT_ST ? 0 : stage + 1;
    const uint32_t next_phase = next == 0 ? phase ^ 1 : phase;
    mbar_wait(&full_bar[next], next_phase);
    // ---- issue S_j = Q K_j^T and O += P_{j-1} V_{j-1} ----
    named_bar_sync(bar_mine, 256);
    reg_fence(o);
    wgmma_fence();
    attn_issue_s<DKC, DVP, BKV>(s, q_base, smem_u32(sK + next * Cfg::K_STAGE));
    attn_issue_pv<DKC, DVP, BKV>(o, pa, smem_u32(sV + stage * Cfg::V_STAGE));
    named_bar_arrive(bar_other, 256);
    // ---- softmax of tile j under the PV product of tile j - 1 ----
    wgmma_wait<1>();
    reg_fence(s);
    softmax(j);
    wgmma_wait<0>();
    reg_fence(o);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
    for (int jb = 0; jb < DVP / 8; ++jb) {
      o[4 * jb + 0] *= corr[0];
      o[4 * jb + 1] *= corr[0];
      o[4 * jb + 2] *= corr[1];
      o[4 * jb + 3] *= corr[1];
    }
    pack_p();
    stage = next;
    phase = next_phase;
  }

  // ---- drain: O += P V of the last tile ----
  named_bar_sync(bar_mine, 256);
  reg_fence(o);
  wgmma_fence();
  attn_issue_pv<DKC, DVP, BKV>(o, pa, smem_u32(sV + stage * Cfg::V_STAGE));
  if (wg == 0) named_bar_arrive(bar_other, 256);  // warpgroup 1 issues last: nobody waits for its arrival
  wgmma_wait<0>();
  reg_fence(o);
  if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);

  // ---- normalise and store ----
  const int q2 = 2 * (lane & 3);
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
