// sdw_gemm.cu — the wgmma implicit-GEMM kernel behind every Conv2d 3x3 / 1x1, Linear and batched matmul of the
// UNet2DCondition / AutoencoderKL-decoder hot path (reference call sites: stable_diffusion_pipeline.py:418
// `self.unet(...)`, :433 `self.vae.decode`).
//
// One CTA computes 128 x (NSUB * BN) output tiles, persistent over a static round-robin of tiles (N fastest, so the
// column tiles of one activation tile run at the same time and the activation tile leaves DRAM once):
//   warps 0-7 : two consumer warpgroups, rows 0-63 / 64-127 of the tile.  Per K block (tap, 64-channel chunk) each
//               issues 4 x wgmma m64nBNk16 per accumulator from the shared-memory ring (fp32 accumulators in registers,
//               one wgmma group kept in flight), then runs the fused epilogue of the tile from its registers:
//               alpha / bias / time-embedding row vector / SiLU / residual / GEGLU / per-head V^T scatter, fp16 out,
//               stored directly (the TMA epilogue's residual arriving per 32-column chunk by TMA into shared
//               memory) or, for GEGLU, staged per 32-column chunk in shared memory and written by TMA stores.
//   warp 8    : TMA producer — per K block one 4-D box of the shifted NHWC activation tile (OOB halo = zero fill =
//               conv padding) and the K-major weight tile(s), SWIZZLE_128B, into an nstages-deep ring.
//
// CL = 2 (the CTA-pair plan): two CTAs of a cluster work on vertically adjacent M tiles with the same weight tile.
// Each loads its own activation rows and HALF of the weight tile, multicast into both CTAs' shared memory, so weight
// bytes per tile fetched from L2 halve; a stage is released only when the consumers of both CTAs are done with it.
//
// TR = 1 (tap reuse, 3x3 stride-1 convs on 16 x 8-pixel tiles): the three ky taps of one kx read the same pixels
// shifted by whole image rows, so one TMA box of (8 + 2) rows x 16 px x 64 ch per (channel chunk, kx) serves three
// taps: tap ky's A operand is the same shared-memory tile entered 16 rows (2 KB, swizzle-atom aligned) further down.
// NSUB = 2: two accumulators per activation tile (128 x 2*BN tiles).
#include "sdw_internal.h"
#include "sdw_ptx.cuh"

#include <cudaTypedefs.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

namespace sdw {

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int GEMM_THREADS = 288;  // two consumer warpgroups + one producer warp
static constexpr int A_STAGE = BM * BK * 2;  // 16 KiB
static constexpr int TR_BW = 16, TR_BH = 8;
static constexpr int A_STAGE_TR = (TR_BH + 2) * TR_BW * 128;  // 20 KiB

template <int BN, int NSUB, int TR>
struct GemmCfg {
  static constexpr int A_BYTES = TR ? A_STAGE_TR : A_STAGE;
  static constexpr int TAPS = TR ? 3 : 1;  // weight tiles (taps) per pipeline stage
  static constexpr int B_SUB = BN * 128;   // one BN-row weight tile
  static constexpr int B_BYTES = TAPS * NSUB * B_SUB;
};

struct EpiRow {
  bool ok;
  int64_t out_off, res_off, pix;
  const float* rowvec;
};

// fused epilogue of one accumulator (columns n_base .. n_base + BN) of this warpgroup's 64 rows.  XE = 1 (the extended
// epilogue of the Real-ESRGAN dense blocks): LeakyReLU(0.2), a scale on the residual and a second, unit-scale residual;
// XE = 0 compiles the original epilogue unchanged.
template <int BN, int XE>
__device__ __forceinline__ void gemm_epilogue(const GemmKParams& p, float (&acc)[BN / 2], int n_base, const EpiRow (&R)[2],
                                              int lane, int wg, int lrow0, uint8_t* stage, uint64_t* res_full, int x0,
                                              int y0, int b0, uint32_t& chunk_count) {
  const int q2 = 2 * (lane & 3);
  const bool vec2 = p.vec2;
  const bool use_tma = p.epi_tma;
  // TMA origin of this warpgroup's 64 rows: a (hw, hh, hb) sub-box of the (bw, bh, bb) tile
  const int r0 = 64 * wg;
  const int tx = x0 + (r0 & (p.bw - 1)), ty = y0 + ((r0 >> p.lg_bw) & (p.bh - 1)), tb = b0 + (r0 >> (p.lg_bw + p.lg_bh));
  const bool issuer = (threadIdx.x & 127) == 0;
  // TMA epilogue with a residual: chunk k's [64 rows x 32 columns] residual arrives by TMA in buffer k & 1, issued one
  // chunk ahead — the first one before this accumulator's first chunk — once every thread of the warpgroup has read
  // the buffer's previous residual chunk (the barrier at the start of each chunk).  Plain outputs leave from registers
  // by direct stores: a TMA store would wait behind the operand loads queued on the same TMA unit, and the chunk loop
  // behind it for its buffer.
  const bool tma_res = use_tma && p.resid != nullptr;
  const int nch = (min(BN, p.N - n_base) + 31) >> 5;
  auto res_issue = [&](int c, uint32_t k) {
    if (tma_res && issuer && c < nch) {
      mbar_expect_tx(&res_full[k & 1], 4096);
      tma_load_4d(&p.mapRes, &res_full[k & 1], stage + (k & 1) * 4096, n_base + 32 * c, tx, ty, tb);
    }
  };
  if (tma_res && p.mode == GEMM_PLAIN) res_issue(0, chunk_count);

  auto value = [&](float v, int n, int h) {
    float o = v * p.alpha;
    if (p.bias) o += __ldg(p.bias + n);
    if (p.rowvec) o += __ldg(R[h].rowvec + n);
    if (p.act == 1) o = silu_f(o);
    if constexpr (XE != 0) {
      if (p.act == 2) o = o > 0.f ? o : 0.2f * o;
    }
    return o;
  };
  auto add_res = [&](float& o, float r) {
    if constexpr (XE != 0) o = fmaf(p.res_scale, r, o);
    else o += r;
  };
  // 2 x 2 values (rows h = 0 / 1, columns n, n + 1) of the plain path, residual added (from the TMA-loaded chunk
  // res_buf, column scol, or from global memory), stored
  auto plain_pair = [&](int j, int n, const uint8_t* res_buf, int scol) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float o0 = n < p.N ? value(acc[4 * j + 2 * h], n, h) : 0.f;
      float o1 = n + 1 < p.N ? value(acc[4 * j + 2 * h + 1], n + 1, h) : 0.f;
      if (res_buf) {
        const float2 f =
            __half22float2(*reinterpret_cast<const __half2*>(res_buf + (lrow0 + 8 * h) * 64 + scol * 2));
        add_res(o0, f.x);
        add_res(o1, f.y);
      } else if (p.resid && R[h].ok) {
        if (vec2 && n + 1 < p.N) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(p.resid + R[h].res_off + n));
          add_res(o0, f.x);
          add_res(o1, f.y);
          if (XE != 0 && p.resid2) {
            const float2 g = __half22float2(*reinterpret_cast<const __half2*>(p.resid2 + R[h].res_off + n));
            o0 += g.x;
            o1 += g.y;
          }
        } else {
          if (n < p.N) add_res(o0, __half2float(p.resid[R[h].res_off + n]));
          if (n + 1 < p.N) add_res(o1, __half2float(p.resid[R[h].res_off + n + 1]));
          if (XE != 0 && p.resid2) {
            if (n < p.N) o0 += __half2float(p.resid2[R[h].res_off + n]);
            if (n + 1 < p.N) o1 += __half2float(p.resid2[R[h].res_off + n + 1]);
          }
        }
      }
      if (R[h].ok) {
        __half* dst = p.out + R[h].out_off + n;
        if (vec2 && n + 1 < p.N) {
          *reinterpret_cast<uint32_t*>(dst) = pack_h2(o0, o1);
        } else {
          if (n < p.N) dst[0] = __float2half_rn(o0);
          if (n + 1 < p.N) dst[1] = __float2half_rn(o1);
        }
      }
    }
  };
  // V^T scatter (columns >= vt_col0): element (b, head, dd, token)
  auto vt_pair = [&](int j, int n) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!R[h].ok) continue;
      const int64_t bq = R[h].pix / p.vt_ntok;
      const int tok = static_cast<int>(R[h].pix - bq * p.vt_ntok);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int nn = n + e;
        if (nn >= p.N) continue;
        float o = acc[4 * j + 2 * h + e] * p.alpha;
        if (p.bias) o += __ldg(p.bias + nn);
        const int cc = nn - p.vt_col0, head = cc / p.vt_d, dd = cc - head * p.vt_d;
        p.vt[((bq * p.vt_heads + head) * p.vt_d + dd) * p.vt_ld + tok] = __float2half_rn(o);
      }
    }
  };
  // staged GEGLU chunk (two 4 KB buffers per warpgroup, alternating): wait until the TMA store that last read the
  // buffer is done, fill it, hand it to the async proxy, store
  auto stage_begin = [&]() {
    if (issuer) bulk_wait_group_read<1>();
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
    return stage + (chunk_count & 1) * 4096;
  };
  auto stage_end = [&](uint8_t* buf, int col) {
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
    if (issuer) {
      tma_store_4d(&p.mapOut, buf, col, tx, ty, tb);
      bulk_commit_group();
    }
    ++chunk_count;
  };

  if (p.mode == GEMM_GEGLU) {
    // packed [32 value | 32 gate] column pairs -> 32 outputs a * gelu(g) per 64 accumulator columns
#pragma unroll
    for (int c = 0; c < BN / 64; ++c) {
      const int n = n_base + 64 * c;
      if (n >= p.N) break;
      uint8_t* buf = use_tma ? stage_begin() : nullptr;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 8 * c + jj;
        const int na = n + 8 * jj + q2, ng = na + 32;
        float o[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float a = acc[4 * j + 2 * h + e] * p.alpha, g = acc[4 * (j + 4) + 2 * h + e] * p.alpha;
            if (p.bias) {
              a += __ldg(p.bias + na + e);
              g += __ldg(p.bias + ng + e);
            }
            o[h][e] = geglu_f(a, g);
          }
        const int ocol = n / 2 + 8 * jj + q2;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (use_tma) {
            *reinterpret_cast<uint32_t*>(buf + (lrow0 + 8 * h) * 64 + (8 * jj + q2) * 2) = pack_h2(o[h][0], o[h][1]);
          } else if (R[h].ok) {
            __half* dst = p.out + R[h].out_off + ocol;
            if (vec2) {
              *reinterpret_cast<uint32_t*>(dst) = pack_h2(o[h][0], o[h][1]);
            } else {
              dst[0] = __float2half_rn(o[h][0]);
              dst[1] = __float2half_rn(o[h][1]);
            }
          }
        }
      }
      if (use_tma) stage_end(buf, n / 2);
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < BN / 32; ++c) {
    const int n = n_base + 32 * c;
    if (n >= p.N) break;
    if (p.mode == GEMM_QKV_VT && n >= p.vt_col0) {  // vt_col0 % 32 == 0: a chunk is all Q|K or all V
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) vt_pair(4 * c + jj, n + 8 * jj + q2);
      continue;
    }
    if (tma_res) {
      // every thread is done with the other buffer (chunk k - 1's residual): generic reads before the async-proxy write
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
      res_issue(c + 1, chunk_count + 1);
      const uint8_t* buf = stage + (chunk_count & 1) * 4096;
      mbar_wait(&res_full[chunk_count & 1], (chunk_count >> 1) & 1);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) plain_pair(4 * c + jj, n + 8 * jj + q2, buf, 8 * jj + q2);
      ++chunk_count;
    } else {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) plain_pair(4 * c + jj, n + 8 * jj + q2, nullptr, 0);
    }
  }
}

template <int BN, int NSUB, int TR, int CL, int XE>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_kernel(const __grid_constant__ GemmKParams p) {
  using Cfg = GemmCfg<BN, NSUB, TR>;
  constexpr int A_BYTES = Cfg::A_BYTES;
  constexpr int B_BYTES = Cfg::B_BYTES;
  const int STAGES = p.nstages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + GEMM_MAX_STAGES;
  uint8_t* smem_a = smem + GEMM_BAR_BYTES;
  uint8_t* smem_b = smem_a + STAGES * A_BYTES;
  uint8_t* epi_stage = smem_b + STAGES * B_BYTES;  // epi_tma: 2 x 4 KB output buffers per consumer warpgroup
  uint64_t* res_full = empty_bar + GEMM_MAX_STAGES;  // [2 warpgroups][2 buffers]: residual chunk arrived

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = CL > 1 ? cluster_ctarank() : 0;
  const int cluster_id = blockIdx.x / CL;
  const int nclusters = gridDim.x / CL;
  const int total_tiles = p.m_groups * p.n_tiles;
  const int num_kb = TR ? 3 * p.kchunks : p.ntaps * p.kchunks;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&p.mapA[0]);
    tma_prefetch_desc(&p.mapB);
    if (p.epi_tma) tma_prefetch_desc(&p.mapOut);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * CL);  // both consumer warpgroups of every CTA that reads the stage's weight halves
    }
    for (int i = 0; i < 4; ++i) mbar_init(&res_full[i], 1);
    if (p.epi_tma && p.resid) tma_prefetch_desc(&p.mapRes);
    fence_barrier_init();
  }
  if (CL > 1) cluster_sync_all();
  else __syncthreads();
  pdl_wait();               // the set-up above overlapped the previous kernel's tail; its outputs are visible from here
  pdl_launch_dependents();

  auto tile_coords = [&](int t, int& x0, int& y0, int& b0, int& n0) {
    const int m_group = t / p.n_tiles;
    const int n_tile = t - m_group * p.n_tiles;
    const int m_tile = m_group * CL + static_cast<int>(rank);
    const int twh = p.tiles_w * p.tiles_h;
    const int tb = m_tile / twh;
    const int rem = m_tile - tb * twh;
    const int th = rem / p.tiles_w;
    const int tw = rem - th * p.tiles_w;
    x0 = tw * p.bw;
    y0 = th * p.bh;
    b0 = tb * p.bb;
    n0 = n_tile * (NSUB * BN);
  };

  if (warp == 8) {
    // =========================== TMA producer ===============================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = cluster_id; t < total_tiles; t += nclusters) {
        int x0, y0, b0, n0;
        tile_coords(t, x0, y0, b0, n0);
        int tap = 0, kc = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], A_BYTES + B_BYTES);  // with CL = 2 half of B arrives from the peer CTA
          uint8_t* a_dst = smem_a + stage * A_BYTES;
          uint8_t* b_dst = smem_b + stage * B_BYTES + rank * (BN / CL) * 128;
          const int nrow = n0 + static_cast<int>(rank) * (BN / CL);
          if (TR) {
            const int kx = tap;  // tap reuse: `tap` counts the column tap kx = 0..2 of channel chunk kc
            tma_load_4d(&p.mapA[0], &full_bar[stage], a_dst, kc * BK, x0 + kx - 1, y0 - 1, b0);
          } else {
            tma_load_4d(&p.mapA[p.tap_map[tap]], &full_bar[stage], a_dst, kc * BK, x0 + p.tap_dx[tap], y0 + p.tap_dy[tap],
                        b0);
          }
#pragma unroll
          for (int ky = 0; ky < Cfg::TAPS; ++ky)
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) {
              const int kcoord = TR ? ((ky * 3 + tap) * p.kchunks + kc) * BK : kb * BK;
              uint8_t* dst = b_dst + (ky * NSUB + sub) * Cfg::B_SUB;
              const int c2 = p.b_batched ? y0 : 0, c3 = p.b_batched ? b0 : 0;
              if (CL > 1)
                tma_load_4d_mc(&p.mapB, &full_bar[stage], dst, kcoord, nrow + sub * BN, c2, c3, (1u << CL) - 1);
              else
                tma_load_4d(&p.mapB, &full_bar[stage], dst, kcoord, nrow + sub * BN, c2, c3);
            }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
          if (TR) {
            if (++tap == 3) {
              tap = 0;
              ++kc;
            }
          } else if (++kc == p.kchunks) {
            kc = 0;
            ++tap;
          }
        }
      }
    }
  } else {
    // =========================== consumers: MMA + epilogue ============================
    const int wg = warp >> 2;
    const int lrow0 = 16 * (warp & 3) + (lane >> 2);  // this thread's first row within the warpgroup's 64
    uint8_t* stage_buf = epi_stage + wg * 8192;
    uint32_t chunk_count = 0;
    // arrival on the empty barrier of `s` in every CTA of the cluster (one thread per warpgroup)
    auto release = [&](int s) {
      if ((threadIdx.x & 127) == 0) {
        if (CL > 1) {
#pragma unroll
          for (int r = 0; r < CL; ++r) mbar_arrive_cluster(mapa_rank(smem_u32(&empty_bar[s]), r));
        } else {
          mbar_arrive(&empty_bar[s]);
        }
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    float acc[NSUB][BN / 2];
    for (int t = cluster_id; t < total_tiles; t += nclusters) {
      int x0, y0, b0, n0;
      tile_coords(t, x0, y0, b0, n0);
#pragma unroll
      for (int sub = 0; sub < NSUB; ++sub)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[sub][i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_base = smem_u32(smem_a + stage * A_BYTES);
        const uint32_t b_base = smem_u32(smem_b + stage * B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int ky = 0; ky < Cfg::TAPS; ++ky) {
          // rows of this warpgroup: 64 lattice points = 4 image rows of the 16-px tap-reuse tile, entered ky rows down
          const uint32_t a_off = TR ? (4 * wg + ky) * (TR_BW * 128) : wg * (64 * 128);
          const uint64_t da = make_desc_k_sw128(a_base + a_off);
#pragma unroll
          for (int k = 0; k < BK / 16; ++k)
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) {
              const uint64_t db = make_desc_k_sw128(b_base + (ky * NSUB + sub) * Cfg::B_SUB);
              Wgmma<BN>::ss(acc[sub], da + 2 * k, db + 2 * k, (kb | ky | k) != 0 ? 1u : 0u);
            }
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous K block's MMAs have read their stage
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int sub = 0; sub < NSUB; ++sub) reg_fence(acc[sub]);
      release(prev);

      // ---- epilogue: rows lrow0 and lrow0 + 8 of this warpgroup ----
      EpiRow R[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = 64 * wg + lrow0 + 8 * h;
        const int x = x0 + (r & (p.bw - 1)), y = y0 + ((r >> p.lg_bw) & (p.bh - 1)), b = b0 + (r >> (p.lg_bw + p.lg_bh));
        R[h].ok = x < p.W && y < p.H && b < p.B;
        R[h].pix = (static_cast<int64_t>(b) * p.H + y) * p.W + x;
        const int64_t oyy = static_cast<int64_t>(y) * p.os + p.oy, oxx = static_cast<int64_t>(x) * p.os + p.ox;
        R[h].out_off = static_cast<int64_t>(b) * p.o_sB + oyy * p.o_sH + oxx * p.o_sW;
        R[h].res_off = static_cast<int64_t>(b) * p.r_sB + oyy * p.r_sH + oxx * p.r_sW;
        R[h].rowvec = p.rowvec ? p.rowvec + static_cast<int64_t>(b) * p.rowvec_ld : nullptr;
      }
#pragma unroll
      for (int sub = 0; sub < NSUB; ++sub)
        gemm_epilogue<BN, XE>(p, acc[sub], n0 + sub * BN, R, lane, wg, lrow0, stage_buf, res_full + 2 * wg, x0, y0, b0,
                          chunk_count);
    }
    if (p.epi_tma && (threadIdx.x & 127) == 0) bulk_wait_group<0>();  // every TMA-stored chunk has reached global memory
  }

  // no CTA of a pair may exit while its peer can still multicast into its shared memory or arrive on its barriers
  if (CL > 1) cluster_sync_all();
}

// =============================================================================
// host side
// =============================================================================
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
static bool g_plan_only = false;  // validate plans without a driver (CPU-side tests); nothing can be launched
void set_plan_only(bool on) { g_plan_only = on; }

int sm_count() {
  static int n = 0;
  if (g_plan_only) return H100_SMS;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        n <= 0) {
      (void)cudaGetLastError();
      n = H100_SMS;
    }
  }
  return n;
}

int gemm_init() {
  if (g_encode || g_plan_only) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  SDW_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || !fn) {
    set_error("cuTensorMapEncodeTiled driver entry point not available");
    return 2;
  }
  g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  return 0;
}

// rank-`rank` fp16 tensor map, dim 0 contiguous, zero OOB fill.
int encode_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
               const uint32_t* box, int swizzle_bytes) {
  if (int e = gemm_init()) return e;
  cuuint64_t gdim[5];
  cuuint64_t gstride[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) {
      gstride[i - 1] = strides_elems[i] * 2;
      if (gstride[i - 1] % 16 != 0) {
        set_error("TMA global stride must be a multiple of 16 bytes");
        return 1;
      }
    }
  }
  if (reinterpret_cast<uintptr_t>(base) % 16 != 0) {
    set_error("TMA global base must be 16-byte aligned");
    return 1;
  }
  for (int i = 0; i < rank; ++i) {
    if (bx[i] == 0 || bx[i] > 256 || gdim[i] == 0) {
      set_error("TMA box dims must be in 1..256 and tensor dims non-zero");
      return 1;
    }
  }
  if (g_plan_only) return 0;
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstride, bx, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_bytes == 0 ? CU_TENSOR_MAP_SWIZZLE_NONE
                                           : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B),
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)));
    return 2;
  }
  return 0;
}

static int pow2_floor(int v) {
  int p = 1;
  while (p * 2 <= v) p *= 2;
  return p;
}

static int stages_for(int bn, int nsub, bool reuse, int epi_bytes) {
  const int a = reuse ? A_STAGE_TR : A_STAGE;
  const int b = (reuse ? 3 : 1) * nsub * bn * 128;
  return std::min(GEMM_MAX_STAGES, (GEMM_SMEM_USABLE - GEMM_BAR_BYTES - epi_bytes) / (a + b));
}

int plan_gemm(const GemmDesc& d, GemmLaunch* L) {
  SDW_REQUIRE(d.A && d.Wt && d.out, "null operand");
  SDW_REQUIRE(d.C > 0 && d.W > 0 && d.H > 0 && d.B > 0 && d.N > 0, "empty problem");
  GemmKParams& p = L->p;
  std::memset(&p, 0, sizeof(p));
  const int kchunks = (d.C + BK - 1) / BK;
  const int Cp = kchunks * BK;
  p.kchunks = kchunks;
  p.ntaps = d.conv == 0 ? 1 : (d.conv == 3 ? 4 : 9);
  // domain (lattice the M tiles walk over) and the tap table
  int Wd = d.W, Hd = d.H;
  int nmaps = 1;
  p.os = 1;
  p.ox = p.oy = 0;
  if (d.conv == 0) {
    p.tap_map[0] = 0;
    p.tap_dx[0] = p.tap_dy[0] = 0;
  } else if (d.conv == 1) {
    for (int t = 0; t < 9; ++t) {
      p.tap_map[t] = 0;
      p.tap_dy[t] = static_cast<int8_t>(t / 3 - 1);
      p.tap_dx[t] = static_cast<int8_t>(t % 3 - 1);
    }
  } else if (d.conv == 2) {
    SDW_REQUIRE(d.W % 2 == 0 && d.H % 2 == 0, "stride-2 conv needs even extents");
    Wd = d.W / 2;
    Hd = d.H / 2;
    nmaps = 4;
    // in = 2*o + k - 1 : k=0 -> parity 1 shift -1 ; k=1 -> parity 0 shift 0 ; k=2 -> parity 1 shift 0
    const int par[3] = {1, 0, 1};
    const int sh[3] = {-1, 0, 0};
    for (int t = 0; t < 9; ++t) {
      const int ky = t / 3, kx = t % 3;
      p.tap_map[t] = static_cast<int8_t>(par[ky] * 2 + par[kx]);
      p.tap_dy[t] = static_cast<int8_t>(sh[ky]);
      p.tap_dx[t] = static_cast<int8_t>(sh[kx]);
    }
  } else if (d.conv == 3) {
    // nearest-up x2 then 3x3, folded into a 2x2 conv per output parity (weights from pack_weight_up4):
    // parity 0 reads low-res rows {yo-1, yo}, parity 1 reads {yo, yo+1}; same for columns
    for (int t = 0; t < 4; ++t) {
      const int a = t >> 1, b = t & 1;
      p.tap_map[t] = 0;
      p.tap_dy[t] = static_cast<int8_t>(d.up_py ? a : a - 1);
      p.tap_dx[t] = static_cast<int8_t>(d.up_px ? b : b - 1);
    }
    p.os = 2;
    p.ox = d.up_px;
    p.oy = d.up_py;
  } else {
    SDW_REQUIRE(false, "unknown conv kind");
  }
  p.W = Wd;
  p.H = Hd;
  p.B = d.B;
  const int64_t OW = static_cast<int64_t>(Wd) * p.os, OH = static_cast<int64_t>(Hd) * p.os;
  // tile geometry: bw*bh*bb = 128
  int bw = std::min(pow2_floor(Wd), BM);
  if (Wd > BM) bw = BM;
  int bh = std::min(pow2_floor(Hd), BM / bw);
  int bb = BM / (bw * bh);
  if (d.b_batched) {
    SDW_REQUIRE(d.conv == 0, "batched matmul is 1x1");
    bw = BM;
    bh = 1;
    bb = 1;
  }
  p.bw = bw;
  p.bh = bh;
  p.bb = bb;
  p.tiles_w = (Wd + bw - 1) / bw;
  p.tiles_h = (Hd + bh - 1) / bh;
  const int tiles_b = (d.B + bb - 1) / bb;
  p.N = d.N;
  p.b_batched = d.b_batched;
  // kernel version: CTA pairs (weight tile multicast to two M tiles) need >= 2 M tiles and a wide-enough N; batched
  // matmuls must pair within one (h, b)
  const int m_tiles = p.tiles_w * p.tiles_h * tiles_b;
  SDW_REQUIRE(d.act >= 0 && d.act <= 2, "activation: 0 none, 1 SiLU, 2 LeakyReLU(0.2)");
  SDW_REQUIRE(!d.resid2 || (d.resid && d.mode == GEMM_PLAIN), "a second residual needs the first one and the plain mode");
  // the extended epilogue (LeakyReLU, residual scale, second residual) and BLOCK_N 32 exist as single-CTA kernels with
  // BLOCK_N 32 / 64 only; every other descriptor plans exactly as before
  const bool xe = d.act == 2 || d.res_scale != 1.f || d.resid2 != nullptr || d.bn == 32;
  L->xe = xe ? 1 : 0;
  if (xe) SDW_REQUIRE(d.ver != 2 && (d.bn == 0 || d.bn == 32 || d.bn == 64) && d.mode == GEMM_PLAIN && d.tr != 2 && d.nsub < 2,
                      "BLOCK_N 32, LeakyReLU and the residual scales need single CTAs with BLOCK_N 32 or 64 (plain mode)");
  int ver = d.ver;
  if (ver == 0 && xe) ver = 1;
  if (ver == 0) ver = (m_tiles >= 2 && d.N >= 128 && (!d.b_batched || p.tiles_w % 2 == 0)) ? 2 : 1;
  SDW_REQUIRE(ver == 1 || ver == 2, "unknown kernel version");
  if (ver == 2) SDW_REQUIRE(!d.b_batched || p.tiles_w % 2 == 0, "CTA-pair batched matmul needs an even tile count per row");
  // tap reuse (3x3 stride 1, CTA pairs): 16 x 8-pixel tiles, one 10-row activation box per (channel chunk, kx)
  bool reuse = false;
  {
    const bool can = ver == 2 && d.conv == 1 && Wd % 16 == 0 && Hd % 8 == 0;
    if (d.tr == 2) SDW_REQUIRE(can, "tap reuse needs a 3x3 stride-1 conv on the CTA-pair kernel with W % 16 == 0, H % 8 == 0");
    reuse = can && d.tr != 1;
    if (reuse) {
      p.bw = bw = TR_BW;
      p.bh = bh = TR_BH;
      p.bb = bb = 1;
      p.tiles_w = Wd / TR_BW;
      p.tiles_h = Hd / TR_BH;
    }
  }
  L->tr = reuse ? 1 : 0;
  const int CL = ver == 2 ? 2 : 1;
  const int nsm = sm_count();
  // ---- epilogue flavour: residual chunks loaded and GEGLU output chunks stored by TMA where the views allow ----
  const int ncols = d.mode == GEMM_GEGLU ? d.N / 2 : (d.mode == GEMM_QKV_VT ? d.vt_col0 : d.N);
  const int64_t osW = d.o_sW || d.o_sH || d.o_sB ? d.o_sW : d.ldc;
  const int64_t osH = d.o_sW || d.o_sH || d.o_sB ? d.o_sH : OW * d.ldc;
  const int64_t osB = d.o_sW || d.o_sH || d.o_sB ? d.o_sB : OH * OW * d.ldc;
  bool can_tma;
  int64_t res_sW, res_sH, res_sB;
  {
    auto ok16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
    auto ok_strides = [&](int64_t sw, int64_t sh, int64_t sb) {
      return sw > 0 && sw % 8 == 0 && (Hd == 1 || sh % 8 == 0) && (d.B == 1 || sb % 8 == 0);
    };
    const bool vt_ok = d.mode != GEMM_QKV_VT || (d.vt_col0 % 32 == 0 && !d.resid);
    const int64_t ldr = d.ldr ? d.ldr : d.ldc;
    const bool rs = d.r_sW || d.r_sH || d.r_sB;
    res_sW = rs ? d.r_sW : ldr;
    res_sH = rs ? d.r_sH : OW * ldr;
    res_sB = rs ? d.r_sB : OH * OW * ldr;
    const bool res_ok = !d.resid || (d.mode == GEMM_PLAIN && !d.resid2 && ok16(d.resid) && ok_strides(res_sW, res_sH, res_sB));
    can_tma = !d.b_batched && vt_ok && res_ok && (!d.rowvec || d.rowvec_ld == 0) && d.N % 8 == 0 && ncols > 0 &&
              ok16(d.out) && ok_strides(osW, osH, osB) && (!d.bias || ok16(d.bias));
    if (d.et == 2) SDW_REQUIRE(can_tma, "the TMA epilogue needs no per-sample row vector and 16-byte aligned views");
    p.epi_tma = can_tma && d.et != 1 ? 1 : 0;
  }
  const int epi_bytes = p.epi_tma ? GEMM_EPI_BYTES : 0;
  // ---- BLOCK_N: wgmma runs 2 x 64 x BN x 16 per instruction at a fixed rate, so a tile's mainloop time grows with its
  // width; the choice minimises waves x tile width (the padded columns of the last N tile included), prefers the wider
  // tile on a tie (fewer activation reloads) and avoids plans that leave fewer than three pipeline stages ----
  int bn = d.bn;
  int nsub = d.nsub ? d.nsub : 1;
  SDW_REQUIRE(nsub == 1 || nsub == 2, "one or two accumulators per activation tile");
  if (nsub == 2) SDW_REQUIRE(ver == 2 && (bn == 0 || bn == 160), "two accumulators: CTA-pair kernel, BLOCK_N 160");
  if (nsub == 2) bn = 160;
  // a tap-reuse stage holds the full weight tiles of three taps: BLOCK_N 256 or two accumulators leave no room for two
  // stages in 227 KB, so the automatic plan falls back to per-tap loads there
  if (reuse && bn && stages_for(bn, nsub, true, epi_bytes) < 2) {
    SDW_REQUIRE(d.tr != 2, "tap reuse with this BLOCK_N / accumulator count does not fit two pipeline stages");
    reuse = false;
    p.bw = bw = std::min(pow2_floor(Wd), BM);
    p.bh = bh = std::min(pow2_floor(Hd), BM / bw);
    p.bb = bb = BM / (bw * bh);
    p.tiles_w = (Wd + bw - 1) / bw;
    p.tiles_h = (Hd + bh - 1) / bh;
    L->tr = 0;
  }
  const int m_tiles_f = p.tiles_w * p.tiles_h * ((d.B + bb - 1) / bb);
  if (bn == 0 && xe) bn = 64;
  if (bn == 0) {
    static const int cand1[4] = {256, 160, 128, 64};
    static const int cand2[4] = {256, 192, 160, 128};
    const int* cand = ver == 2 ? cand2 : cand1;
    double best = 1e30;
    const int groups = (m_tiles_f + CL - 1) / CL;
    for (int i = 0; i < 4; ++i) {
      const int c = cand[i];
      if (d.mode == GEMM_GEGLU && c % 64 != 0) continue;
      if (stages_for(c, 1, reuse, epi_bytes) < 2) continue;
      const int tiles = groups * ((d.N + c - 1) / c);
      const int waves = (tiles + nsm / CL - 1) / (nsm / CL);
      double cost = static_cast<double>(waves) * c;
      if (stages_for(c, 1, reuse, epi_bytes) < 3) cost *= 1.6;  // H100: two-stage tap-reuse plans measured ~1.3-1.5x slower per column
      if (cost < best) {
        best = cost;
        bn = c;
      }
    }
  }
  SDW_REQUIRE(bn == 32 || bn == 64 || bn == 128 || bn == 160 || bn == 256 || (bn == 192 && ver == 2), "unsupported BLOCK_N");
  if (ver == 2) SDW_REQUIRE(bn != 32 && bn != 64, "the CTA-pair kernel needs BLOCK_N >= 128");
  if (d.ew == 4) SDW_REQUIRE(false, "one epilogue form on this GPU: epilogue width 4 is not available");
  SDW_REQUIRE(d.ew == 0 || d.ew == 2, "epilogue width must be 0 (auto) or 2");
  L->ew = 2;
  L->ver = ver;
  L->nsub = nsub;
  L->bn = bn;
  if (d.mode == GEMM_GEGLU) SDW_REQUIRE(bn % 64 == 0 && d.N % 64 == 0, "GEGLU needs 64-column pairs");
  if (d.mode == GEMM_QKV_VT) SDW_REQUIRE(d.vt && d.vt_col0 % 32 == 0 && d.vt_d > 0, "bad V^T split");
  p.nstages = stages_for(bn, nsub, reuse, epi_bytes);
  SDW_REQUIRE(p.nstages >= 2, "no room for a two-stage operand pipeline");
  p.m_groups = (m_tiles_f + CL - 1) / CL;
  p.n_tiles = (d.N + bn * nsub - 1) / (bn * nsub);
  {
    const int64_t total = static_cast<int64_t>(p.m_groups) * p.n_tiles;
    SDW_REQUIRE(total < (int64_t(1) << 31), "tile grid too large");
    L->grid = dim3(static_cast<unsigned>(CL * std::min<int64_t>(total, nsm / CL)), 1, 1);  // persistent
  }
  {
    auto lg2 = [](int v) { int l = 0; while ((1 << l) < v) ++l; return l; };
    p.lg_bw = lg2(p.bw);
    p.lg_bh = lg2(p.bh);
    SDW_REQUIRE((1 << p.lg_bw) == p.bw && (1 << p.lg_bh) == p.bh, "tile extents must be powers of two");
  }
  // tensor maps: A
  for (int m = 0; m < nmaps; ++m) {
    const __half* base = d.A;
    uint64_t dims[4] = {static_cast<uint64_t>(d.C), static_cast<uint64_t>(d.W), static_cast<uint64_t>(d.H),
                        static_cast<uint64_t>(d.B)};
    uint64_t strides[4] = {1, static_cast<uint64_t>(d.sW), static_cast<uint64_t>(d.sH), static_cast<uint64_t>(d.sB)};
    if (d.conv == 2) {
      const int py = m / 2, px = m % 2;
      base = d.A + py * d.sH + px * d.sW;
      dims[1] = Wd;
      dims[2] = Hd;
      strides[1] = 2 * d.sW;
      strides[2] = 2 * d.sH;
    }
    // degenerate extents still need a non-zero, 16B-multiple stride
    for (int i = 1; i < 4; ++i)
      if (strides[i] == 0) strides[i] = static_cast<uint64_t>(Cp);
    uint32_t box[4] = {BK, static_cast<uint32_t>(bw), static_cast<uint32_t>(reuse ? bh + 2 : bh), static_cast<uint32_t>(bb)};
    if (int e = encode_map(&p.mapA[m], base, 4, dims, strides, box)) return e;
  }
  {
    const int64_t ldb = d.ldb ? d.ldb : static_cast<int64_t>(p.ntaps) * Cp;
    uint64_t dims[4] = {static_cast<uint64_t>(d.Kb ? d.Kb : static_cast<int64_t>(p.ntaps) * Cp),
                        static_cast<uint64_t>(d.N), static_cast<uint64_t>(d.b_batched ? Hd : 1),
                        static_cast<uint64_t>(d.b_batched ? d.B : 1)};
    uint64_t strides[4] = {1, static_cast<uint64_t>(ldb), static_cast<uint64_t>(d.b_batched ? d.sBh : 0),
                           static_cast<uint64_t>(d.b_batched ? d.sBb : 0)};
    for (int i = 2; i < 4; ++i)
      if (strides[i] == 0) strides[i] = static_cast<uint64_t>(ldb);
    uint32_t box[4] = {BK, static_cast<uint32_t>(bn / CL), 1, 1};
    if (int e = encode_map(&p.mapB, d.Wt, 4, dims, strides, box)) return e;
  }
  if (p.epi_tma) {
    // output lattice: column, then the tile lattice (w, h, b) with the parity scatter folded into base + strides; the
    // box is one consumer warpgroup's 64 rows x 32 columns
    const int hw = std::min(bw, 64), hh = std::min(bh, 64 / hw), hb = 64 / (hw * hh);
    uint64_t dims[4] = {static_cast<uint64_t>(ncols), static_cast<uint64_t>(Wd), static_cast<uint64_t>(Hd),
                        static_cast<uint64_t>(d.B)};
    uint64_t so[4] = {1, static_cast<uint64_t>(osW * p.os), static_cast<uint64_t>(osH * p.os), static_cast<uint64_t>(osB)};
    for (int i = 2; i < 4; ++i)  // extents of one still need a legal stride
      if (so[i] == 0 || so[i] % 8 != 0) so[i] = so[1] * static_cast<uint64_t>(Wd);
    uint32_t box[4] = {32, static_cast<uint32_t>(hw), static_cast<uint32_t>(hh), static_cast<uint32_t>(hb)};
    if (int e = encode_map(&p.mapOut, d.out + p.oy * osH + p.ox * osW, 4, dims, so, box, 0)) return e;
    if (d.resid) {
      uint64_t sr[4] = {1, static_cast<uint64_t>(res_sW * p.os), static_cast<uint64_t>(res_sH * p.os),
                        static_cast<uint64_t>(res_sB)};
      for (int i = 2; i < 4; ++i)
        if (sr[i] == 0 || sr[i] % 8 != 0) sr[i] = sr[1] * static_cast<uint64_t>(Wd);
      if (int e = encode_map(&p.mapRes, d.resid + p.oy * res_sH + p.ox * res_sW, 4, dims, sr, box, 0)) return e;
    }
  }
  p.bias = d.bias;
  p.rowvec = d.rowvec;
  p.rowvec_ld = d.rowvec_ld;
  p.resid = d.resid;
  p.res_scale = d.res_scale;
  p.resid2 = d.resid2;
  p.out = d.out;
  p.o_sW = osW;
  p.o_sH = osH;
  p.o_sB = osB;
  p.r_sW = res_sW;
  p.r_sH = res_sH;
  p.r_sB = res_sB;
  // two-column (4-byte) output / residual accesses: every row offset and the column pair start even
  p.vec2 = ((p.o_sW | p.o_sH | p.o_sB) & 1) == 0 && (reinterpret_cast<uintptr_t>(d.out) & 3) == 0 &&
           (!d.resid || (((p.r_sW | p.r_sH | p.r_sB) & 1) == 0 && (reinterpret_cast<uintptr_t>(d.resid) & 3) == 0)) &&
           (!d.resid2 || (reinterpret_cast<uintptr_t>(d.resid2) & 3) == 0);
  p.mode = d.mode;
  p.act = d.act;
  p.alpha = d.alpha;
  p.vt_col0 = d.vt_col0;
  p.vt_d = d.vt_d;
  p.vt_heads = d.vt_heads;
  p.vt_ntok = d.vt_ntok > 0 ? d.vt_ntok : 1;
  p.vt = d.vt;
  p.vt_ld = d.vt_ld;
  return 0;
}

template <int BN, int NSUB, int TR, int CL, int XE = 0>
static int launch_one(const GemmLaunch& l, cudaStream_t stream) {
  static int max_ctas = 0;  // CTAs of this kernel that can be resident at once (whole clusters)
  if (!max_ctas) {
    SDW_CUDA_OK(cudaFuncSetAttribute(gemm_kernel<BN, NSUB, TR, CL, XE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     GEMM_SMEM_DYN));
    max_ctas = sm_count();
    if (CL > 1) {
      // clusters must fit inside one GPC: fewer than SMs / CL of them may be co-resident, and a persistent grid larger
      // than that would run its last clusters as a second wave
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3(CL * (sm_count() / CL));
      cfg.blockDim = dim3(GEMM_THREADS);
      cfg.dynamicSmemBytes = GEMM_SMEM_DYN;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = CL;
      attr[0].val.clusterDim.y = 1;
      attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
      int nclusters = 0;
      SDW_CUDA_OK(cudaOccupancyMaxActiveClusters(&nclusters, gemm_kernel<BN, NSUB, TR, CL, XE>, &cfg));
      if (nclusters > 0) max_ctas = std::min(max_ctas, CL * nclusters);
    }
  }
  const dim3 grid(std::min<unsigned>(l.grid.x, static_cast<unsigned>(max_ctas)), 1, 1);
  SDW_CUDA_OK(launch_cluster(gemm_kernel<BN, NSUB, TR, CL, XE>, grid, dim3(GEMM_THREADS), GEMM_SMEM_DYN, stream, CL, l.p));
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

// instantiations: single CTAs with BLOCK_N 64 / 128 / 160 / 256, and BLOCK_N 32 / 64 with the extended epilogue; CTA pairs with BLOCK_N 128 / 160 / 192 / 256 x
// {per-tap, tap reuse} and one accumulator, 160 x 2 accumulators
int launch_gemm(const GemmLaunch& l, cudaStream_t stream) {
  const int key = l.xe * 1000000 + l.ver * 100000 + l.bn * 100 + l.nsub * 10 + (l.tr ? 1 : 0);
  switch (key) {
    case 1103210: return launch_one<32, 1, 0, 1, 1>(l, stream);
    case 1106410: return launch_one<64, 1, 0, 1, 1>(l, stream);
    case 106410: return launch_one<64, 1, 0, 1>(l, stream);
    case 112810: return launch_one<128, 1, 0, 1>(l, stream);
    case 116010: return launch_one<160, 1, 0, 1>(l, stream);
    case 125610: return launch_one<256, 1, 0, 1>(l, stream);
    case 212810: return launch_one<128, 1, 0, 2>(l, stream);
    case 216010: return launch_one<160, 1, 0, 2>(l, stream);
    case 219210: return launch_one<192, 1, 0, 2>(l, stream);
    case 225610: return launch_one<256, 1, 0, 2>(l, stream);
    case 216020: return launch_one<160, 2, 0, 2>(l, stream);
    case 212811: return launch_one<128, 1, 1, 2>(l, stream);
    case 216011: return launch_one<160, 1, 1, 2>(l, stream);
    case 219211: return launch_one<192, 1, 1, 2>(l, stream);
    case 225611: return launch_one<256, 1, 1, 2>(l, stream);
    case 216021: return launch_one<160, 2, 1, 2>(l, stream);
    default: break;
  }
  set_error("no GEMM kernel for this version / BLOCK_N / accumulators / tap reuse combination");
  return 1;
}

}  // namespace sdw
