// sdw_esrgan.cu — the Real-ESRGAN x4 upsampler behind `walk(upsample=True)` / `make_clip_frames(upsample=True)`
// (reference stable_diffusion_pipeline.py:513-516, 550-553 and upsampling.py `RealESRGANModel`): RRDBNet x4
// (basicsr: 64 features, `num_block` RRDBs, 32 growth channels) on 8-bit RGB frames, natively.
//
//   conv_first   uint8 RGB -> fp16(u / 255) -> 3x3, 3 -> 64                    (CUDA cores, sdw_norm.cu conv_in_kernel)
//   body         num_block x RRDB; RDB: x1..x4 = lrelu(conv_k(cat(x, x1..x_{k-1}))), 64/96/128/160 -> 32,
//                x5 = conv5(cat(...)) 192 -> 64, rdb(x) = 0.2 x5 + x; RRDB(x) = 0.2 rdb3(rdb2(rdb1(x))) + x
//   conv_body    64 -> 64, + feat
//   conv_up1/2   nearest x2 + 3x3 + lrelu, folded into four 2x2 parity convs (pack_weight_up4)
//   conv_hr      3x3 + lrelu;  conv_last 64 -> 3, round(clamp(v, 0, 1) * 255)   (CUDA cores, conv_out_kernel)
// Every 3x3 conv except the two edge ones runs on the wgmma implicit GEMM of sdw_gemm.cu.
//
// A dense block lives in one 192-channel NHWC buffer: slice [0, 64) is the block input, conv_k writes its 32-channel
// slice [32 (k + 1), 32 (k + 2)) straight from the GEMM epilogue, and conv5 reads all 192 channels (the reads of
// conv2 / conv4 stop at C = 96 / 160: the tensor map's channel extent is C, TMA zero-fills the rest of the 64-channel
// chunk) and writes the next block's input slice.  The residual scales are folded into the epilogue: conv5 of rdb1 / rdb2
// writes 0.2 (acc + b) + x, conv5 of rdb3 writes 0.04 (acc + b) + 0.2 r + x_rrdb in fp32 before its single rounding
// (biases pre-scaled at load, since alpha multiplies the accumulator before the bias is added).
//
// Memory, by build-time liveness (two regions of one 2048^2 x 64 fp16 map each per 512^2 frame):
//   P: the five 192-channel block buffers X0 X1 X2 Bc Cc of the trunk, later the 4H x 4W map of conv_up2
//   Q: the trunk output t and the 2H x 2W map of conv_up1, later the 4H x 4W map of conv_hr
// X0 holds conv_first's output (`feat`) for the whole trunk; the RRDB chain alternates X1 / X2.
// State-dict names are basicsr's RRDBNet keys (conv_first.*, body.{i}.rdb{1,2,3}.conv{1..5}.*, conv_body.*,
// conv_up1.*, conv_up2.*, conv_hr.*, conv_last.*).
#include "sdw_internal.h"

#include <algorithm>
#include <cstdio>
#include <functional>
#include <string>
#include <vector>

#include "../../include/sdwalk.h"

namespace sdw {

namespace {

struct EsrConv {
  __half* w = nullptr;
  float* b = nullptr;
};

struct EsrEngine {
  sdw_upsampler_config cfg;
  Arena arena{256};
  size_t cap = 0;
  ParamTable params;
  EsrConv first, body_conv, up1, up2, hr, last;
  std::vector<EsrConv> body;  // [block][rdb][conv]: index (i * 3 + r) * 5 + k
  uint8_t *P = nullptr, *Q = nullptr;
  __half *X[3] = {nullptr, nullptr, nullptr}, *Bc = nullptr, *Cc = nullptr, *t = nullptr, *u1 = nullptr, *u2 = nullptr,
         *h = nullptr;
  OpList gemms;  // the static GEMM sequence between conv_first and conv_last, planned at bind time
  GraphCache graph;

  static int64_t cp(int C) { return (C + 63) / 64 * 64; }
  EsrConv conv3(const std::string& name, int N, int C, float bias_scale = 1.f) {
    EsrConv c;
    c.w = arena.take<__half>(static_cast<size_t>(N) * 9 * cp(C));
    c.b = arena.take<float>(N);
    params.add(name + ".weight", PACKED, c.w, static_cast<int64_t>(N) * C * 9, N, C, 3, 3);
    params.add(name + ".bias", VEC, c.b, N, N, 0, 1, 1, 0, bias_scale);
    return c;
  }
  EsrConv conv_up(const std::string& name, int N, int C) {
    EsrConv c;
    c.w = arena.take<__half>(static_cast<size_t>(4) * N * 4 * cp(C));
    c.b = arena.take<float>(N);
    params.add(name + ".weight", PACKED_UP4, c.w, static_cast<int64_t>(N) * C * 9, N, C);
    params.add(name + ".bias", VEC, c.b, N);
    return c;
  }
  EsrConv conv_raw(const std::string& name, int N, int C) {
    EsrConv c;
    c.w = arena.take<__half>(static_cast<size_t>(N) * C * 9);
    c.b = arena.take<float>(N);
    params.add(name + ".weight", RAW, c.w, static_cast<int64_t>(N) * C * 9);
    params.add(name + ".bias", VEC, c.b, N);
    return c;
  }
  int64_t pix() const { return static_cast<int64_t>(cfg.frames) * cfg.in_h * cfg.in_w; }
  void layout(void* base) {
    const int nf = cfg.num_feat, gc = cfg.num_grow_ch;
    arena.reset(base);
    params.clear(base != nullptr);
    body.assign(static_cast<size_t>(cfg.num_block) * 15, EsrConv{});
    first = conv_raw("conv_first", nf, 3);
    for (int i = 0; i < cfg.num_block; ++i)
      for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 5; ++k) {
          const std::string nm = "body." + std::to_string(i) + ".rdb" + std::to_string(r + 1) + ".conv" + std::to_string(k + 1);
          const int C = nf + gc * k;
          body[(i * 3 + r) * 5 + k] = k < 4 ? conv3(nm, gc, C) : conv3(nm, nf, C, r < 2 ? 0.2f : 0.04f);
        }
    body_conv = conv3("conv_body", nf, nf);
    up1 = conv_up("conv_up1", nf, nf);
    up2 = conv_up("conv_up2", nf, nf);
    hr = conv3("conv_hr", nf, nf);
    last = conv_raw("conv_last", 3, nf);
    // activations (see the header): P = max(five block buffers, the 4H x 4W map), Q = max(t + 2H x 2W map, 4H x 4W map)
    const int cat = nf + 4 * gc;  // 192
    const size_t catb = ((static_cast<size_t>(pix()) * cat * 2 + 255) & ~size_t(255));
    const size_t big = ((static_cast<size_t>(pix()) * 16 * nf * 2 + 255) & ~size_t(255));
    const size_t tb = ((static_cast<size_t>(pix()) * nf * 2 + 255) & ~size_t(255));
    const size_t u1b = ((static_cast<size_t>(pix()) * 4 * nf * 2 + 255) & ~size_t(255));
    P = arena.take<uint8_t>(std::max(5 * catb, big));
    Q = arena.take<uint8_t>(std::max(tb + u1b, big));
    if (base) {
      for (int j = 0; j < 3; ++j) X[j] = reinterpret_cast<__half*>(P + j * catb);
      Bc = reinterpret_cast<__half*>(P + 3 * catb);
      Cc = reinterpret_cast<__half*>(P + 4 * catb);
      u2 = reinterpret_cast<__half*>(P);
      t = reinterpret_cast<__half*>(Q);
      u1 = reinterpret_cast<__half*>(Q + tb);
      h = reinterpret_cast<__half*>(Q);
    }
  }

  // one 3x3 (conv = 1) or folded nearest-up x2 + 3x3 parity (conv = 3) GEMM on an NHWC lattice with channel pitch lda
  GemmDesc desc(const __half* A, int C, int64_t lda, int W, int H, const __half* Wt, int N, const float* b, __half* out,
                int64_t ldc, int act) const {
    GemmDesc d;
    d.A = A; d.C = C; d.W = W; d.H = H; d.B = cfg.frames;
    d.sW = lda; d.sH = static_cast<int64_t>(W) * lda; d.sB = static_cast<int64_t>(H) * W * lda;
    d.conv = 1;
    d.Wt = Wt; d.N = N; d.bias = b; d.out = out; d.ldc = ldc; d.act = act;
    return d;
  }
  int build_ops() {
    gemms.clear();
    const int nf = cfg.num_feat, gc = cfg.num_grow_ch, cat = nf + 4 * gc;
    const int W = cfg.in_w, H = cfg.in_h;
    int cur = 0;  // X[cur] holds the RRDB input; X[0] = feat stays untouched
    for (int i = 0; i < cfg.num_block; ++i) {
      const int nxt = cur == 1 ? 2 : 1;
      __half* bufs[4] = {X[cur], Bc, Cc, X[nxt]};
      for (int r = 0; r < 3; ++r) {
        __half* in = bufs[r];
        const std::string pre = "body." + std::to_string(i) + ".rdb" + std::to_string(r + 1) + ".";
        for (int k = 0; k < 4; ++k) {
          const EsrConv& c = body[(i * 3 + r) * 5 + k];
          GemmDesc d = desc(in, nf + gc * k, cat, W, H, c.w, gc, c.b, in + nf + gc * k, cat, 2);
          d.bn = 32;
          d.ver = 1;
          const std::string tag = pre + "conv" + std::to_string(k + 1) + " " + std::to_string(nf + gc * k) + "->32 lrelu";
          if (int e = gemms.add_gemm(d, tag)) return e;
        }
        const EsrConv& c5 = body[(i * 3 + r) * 5 + 4];
        GemmDesc d = desc(in, cat, cat, W, H, c5.w, nf, c5.b, bufs[r + 1], cat, 0);
        d.resid = in;
        d.ldr = cat;
        if (r < 2) {
          d.alpha = 0.2f;
        } else {
          d.alpha = 0.04f;
          d.res_scale = 0.2f;
          d.resid2 = X[cur];
        }
        if (int e = gemms.add_gemm(d, pre + "conv5 192->64" + (r < 2 ? " x0.2 + x" : " x0.04 + 0.2 r + x_rrdb"))) return e;
      }
      cur = nxt;
    }
    {
      GemmDesc d = desc(X[cur], nf, cat, W, H, body_conv.w, nf, body_conv.b, t, nf, 0);
      d.resid = X[0];
      d.ldr = cat;
      if (int e = gemms.add_gemm(d, "conv_body + feat")) return e;
    }
    const __half* src[2] = {t, u1};
    __half* dst[2] = {u1, u2};
    const EsrConv* ups[2] = {&up1, &up2};
    for (int s = 0; s < 2; ++s)
      for (int par = 0; par < 4; ++par) {
        const int py = par >> 1, px = par & 1;
        GemmDesc d = desc(src[s], nf, nf, W << s, H << s, ups[s]->w + static_cast<int64_t>(par) * nf * 4 * cp(nf), nf,
                          ups[s]->b, dst[s], nf, 2);
        d.conv = 3;
        d.up_px = px;
        d.up_py = py;
        const std::string tag = std::string("conv_up") + char('1' + s) + " parity " + char('0' + py) + char('0' + px) + " lrelu";
        if (int e = gemms.add_gemm(d, tag)) return e;
      }
    GemmDesc d = desc(u2, nf, nf, 4 * W, 4 * H, hr.w, nf, hr.b, h, nf, 2);
    return gemms.add_gemm(d, "conv_hr lrelu");
  }
};

}  // namespace
}  // namespace sdw

using namespace sdw;

extern "C" {

int sdw_conv_first_u8(const uint8_t* x, int B, int H, int W, const void* w, const float* bias, int N, void* y, int64_t ldy,
                      void* stream) {
  return conv_first_u8(x, B, H, W, static_cast<const __half*>(w), bias, N, static_cast<__half*>(y), ldy,
                       static_cast<cudaStream_t>(stream));
}

int sdw_conv_last_u8(const void* x, int64_t ldx, int B, int H, int W, int C, const void* w, const float* bias,
                     float* out_f32, uint8_t* out_u8, void* stream) {
  return conv_out_small(static_cast<const __half*>(x), ldx, B, H, W, C, static_cast<const __half*>(w), bias, 3, out_f32,
                        out_u8, static_cast<cudaStream_t>(stream), 1);
}

int sdw_upsampler_create(const sdw_upsampler_config* cfg, sdw_upsampler** out) {
  SDW_REQUIRE(cfg && out, "null");
  SDW_REQUIRE(cfg->num_feat == 64 && cfg->num_grow_ch == 32, "Real-ESRGAN x4: num_feat 64 and num_grow_ch 32 only");
  SDW_REQUIRE(cfg->num_block >= 1 && cfg->num_block <= 64, "num_block in 1..64");
  SDW_REQUIRE(cfg->in_h >= 1 && cfg->in_w >= 1 && cfg->frames >= 1, "bad sizes");
  SDW_REQUIRE(static_cast<int64_t>(cfg->in_h) * cfg->in_w * cfg->frames * 16 < (int64_t(1) << 31), "output too large");
  EsrEngine* E = new EsrEngine();
  E->cfg = *cfg;
  E->layout(nullptr);
  E->cap = E->arena.off;
  *out = reinterpret_cast<sdw_upsampler*>(E);
  return 0;
}

void sdw_upsampler_destroy(sdw_upsampler* e) { delete reinterpret_cast<EsrEngine*>(e); }

int sdw_upsampler_arena_bytes(const sdw_upsampler* e, uint64_t* bytes) {
  const EsrEngine* E = reinterpret_cast<const EsrEngine*>(e);
  SDW_REQUIRE(E && bytes, "null");
  *bytes = E->cap + 256;
  return 0;
}

int sdw_upsampler_bind(sdw_upsampler* e, void* arena, uint64_t bytes) {
  EsrEngine* E = reinterpret_cast<EsrEngine*>(e);
  SDW_REQUIRE(E && arena, "null");
  SDW_REQUIRE(bytes >= E->cap + 256, "arena too small");
  SDW_REQUIRE((reinterpret_cast<uintptr_t>(arena) & 255) == 0, "arena must be 256-byte aligned");
  E->graph.reset();
  E->layout(arena);
  return E->build_ops();
}

int sdw_upsampler_num_params(const sdw_upsampler* e) {
  return e ? reinterpret_cast<const EsrEngine*>(e)->params.size() : 0;
}

int sdw_upsampler_param_info(const sdw_upsampler* e, int index, const char** name, int64_t* numel) {
  SDW_REQUIRE(e, "null");
  return reinterpret_cast<const EsrEngine*>(e)->params.info(index, name, numel);
}

int sdw_upsampler_load_param(sdw_upsampler* e, const char* name, const void* src_f16, int64_t numel, void* stream) {
  SDW_REQUIRE(e, "null");
  return reinterpret_cast<EsrEngine*>(e)->params.load(name, src_f16, numel, static_cast<cudaStream_t>(stream));
}

int sdw_upsampler_missing_params(const sdw_upsampler* e, const char** first_missing) {
  return e ? reinterpret_cast<const EsrEngine*>(e)->params.missing(first_missing) : -1;
}

int sdw_upsampler_run(sdw_upsampler* e, const uint8_t* in_u8, uint8_t* out_u8, float* out_preclamp_f32, int use_graph,
                      void* stream) {
  EsrEngine* E = reinterpret_cast<EsrEngine*>(e);
  SDW_REQUIRE(E && in_u8 && out_u8 && E->params.bound, "null / engine not bound");
  SDW_REQUIRE(E->params.missing(nullptr) == 0, "upsampler parameters not loaded");
  const sdw_upsampler_config& c = E->cfg;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDW_REQUIRE(!use_graph || st != nullptr, "graph capture needs a real stream, not the legacy default stream 0");
  // the edge convs read / write the caller's buffers directly; the GEMM sequence in between works on the arena only and
  // is what the CUDA graph holds
  if (int rc = conv_first_u8(in_u8, c.frames, c.in_h, c.in_w, E->first.w, E->first.b, c.num_feat, E->X[0],
                             c.num_feat + 4 * c.num_grow_ch, st))
    return rc;
  if (use_graph) {
    if (int rc = E->graph.launch(0, st, [E](cudaStream_t s) { return E->gemms.run(s, 0); })) return rc;
  } else {
    if (int rc = E->gemms.run(st, 0)) return rc;
  }
  return conv_out_small(E->h, c.num_feat, c.frames, 4 * c.in_h, 4 * c.in_w, c.num_feat, E->last.w, E->last.b, 3,
                        out_preclamp_f32, out_u8, st, 1);
}

// tooling: CUDA-event time of every op of one forward after one untimed pass, written as "upsampler<TAB>index<TAB>
// microseconds<TAB>tag" lines.  The edge convs read / write dead arena regions here (their values do not matter).
int sdw_upsampler_debug_profile(sdw_upsampler* e, const char* path, void* stream) {
  EsrEngine* E = reinterpret_cast<EsrEngine*>(e);
  SDW_REQUIRE(E && path && E->params.bound, "engine not bound");
  SDW_REQUIRE(E->params.missing(nullptr) == 0, "upsampler parameters not loaded");
  const sdw_upsampler_config& c = E->cfg;
  const uint8_t* in_scratch = E->Q;  // dead while conv_first runs
  uint8_t* out_scratch = E->P;       // dead while conv_last runs
  OpList ops;
  ops.add("conv_first u8 3->64 (CUDA cores)", [=](cudaStream_t st, int) {
    return conv_first_u8(in_scratch, c.frames, c.in_h, c.in_w, E->first.w, E->first.b, c.num_feat, E->X[0],
                         c.num_feat + 4 * c.num_grow_ch, st);
  });
  ops.append(E->gemms);
  ops.add("conv_last 64->3 + uint8 (CUDA cores)", [=](cudaStream_t st, int) {
    return conv_out_small(E->h, c.num_feat, c.frames, 4 * c.in_h, 4 * c.in_w, c.num_feat, E->last.w, E->last.b, 3,
                          nullptr, out_scratch, st, 1);
  });
  FILE* f = std::fopen(path, "w");
  SDW_REQUIRE(f, "cannot open the profile file");
  int rc = profile_ops(f, "upsampler", ops, static_cast<cudaStream_t>(stream), 0);
  std::fclose(f);
  if (rc) return rc;
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
