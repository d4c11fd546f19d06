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
#include <map>
#include <string>
#include <vector>

#include "../../include/sdwalk.h"

namespace sdw {

__global__ void esr_bias_kernel(const __half* __restrict__ in, float* __restrict__ out, int n, float scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __half2float(in[i]) * scale;
}

namespace {

enum EsrKind : int { K_BIAS = 0, K_CONV3 = 1, K_UP4 = 2, K_RAW = 3 };

struct EsrParam {
  void* dst = nullptr;
  int64_t numel = 0;
  int kind = 0;
  int N = 0, C = 0;
  float scale = 1.f;  // biases of conv5: 0.2 (rdb1, rdb2) or 0.04 (rdb3)
  bool loaded = false;
};

struct EsrConv {
  __half* w = nullptr;
  float* b = nullptr;
};

struct EsrEngine {
  sdw_upsampler_config cfg;
  bool dry = true;
  uint8_t* base = nullptr;
  size_t used = 0, cap = 0;
  std::map<std::string, EsrParam> params;
  std::vector<std::string> order;
  EsrConv first, body_conv, up1, up2, hr, last;
  std::vector<EsrConv> body;  // [block][rdb][conv]: index (i * 3 + r) * 5 + k
  uint8_t *P = nullptr, *Q = nullptr;
  __half *X[3] = {nullptr, nullptr, nullptr}, *Bc = nullptr, *Cc = nullptr, *t = nullptr, *u1 = nullptr, *u2 = nullptr,
         *h = nullptr;
  std::vector<GemmLaunch> gemms;  // the static op list between conv_first and conv_last, planned at bind time
  std::vector<std::string> tags;
  cudaGraphExec_t graph_exec = nullptr;

  template <typename T>
  T* take(size_t n) {
    used = (used + 255) & ~size_t(255);
    T* p = dry ? nullptr : reinterpret_cast<T*>(base + used);
    used += n * sizeof(T);
    return p;
  }
  void reg(const std::string& name, void* dst, int64_t numel, int kind, int N = 0, int C = 0, float scale = 1.f) {
    EsrParam p;
    p.dst = dst; p.numel = numel; p.kind = kind; p.N = N; p.C = C; p.scale = scale;
    if (!params.count(name)) order.push_back(name);
    params[name] = p;
  }
  static int64_t cp(int C) { return (C + 63) / 64 * 64; }
  EsrConv conv3(const std::string& name, int N, int C, float bias_scale = 1.f) {
    EsrConv c;
    c.w = take<__half>(static_cast<size_t>(N) * 9 * cp(C));
    c.b = take<float>(N);
    reg(name + ".weight", c.w, static_cast<int64_t>(N) * C * 9, K_CONV3, N, C);
    reg(name + ".bias", c.b, N, K_BIAS, N, 0, bias_scale);
    return c;
  }
  EsrConv conv_up(const std::string& name, int N, int C) {
    EsrConv c;
    c.w = take<__half>(static_cast<size_t>(4) * N * 4 * cp(C));
    c.b = take<float>(N);
    reg(name + ".weight", c.w, static_cast<int64_t>(N) * C * 9, K_UP4, N, C);
    reg(name + ".bias", c.b, N, K_BIAS, N);
    return c;
  }
  EsrConv conv_raw(const std::string& name, int N, int C) {
    EsrConv c;
    c.w = take<__half>(static_cast<size_t>(N) * C * 9);
    c.b = take<float>(N);
    reg(name + ".weight", c.w, static_cast<int64_t>(N) * C * 9, K_RAW, N, C);
    reg(name + ".bias", c.b, N, K_BIAS, N);
    return c;
  }
  int64_t pix() const { return static_cast<int64_t>(cfg.frames) * cfg.in_h * cfg.in_w; }
  void layout() {
    const int nf = cfg.num_feat, gc = cfg.num_grow_ch;
    used = 0;
    params.clear();
    order.clear();
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
    P = take<uint8_t>(std::max(5 * catb, big));
    Q = take<uint8_t>(std::max(tb + u1b, big));
    if (!dry) {
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
  int add(const GemmDesc& d, const std::string& tag) {
    GemmLaunch L;
    if (int e = plan_gemm(d, &L)) {
      set_error(tag + ": " + last_error());
      return e;
    }
    gemms.push_back(L);
    tags.push_back(tag);
    return 0;
  }
  int build_ops() {
    gemms.clear();
    tags.clear();
    const int nf = cfg.num_feat, gc = cfg.num_grow_ch, cat = nf + 4 * gc;
    const int W = cfg.in_w, H = cfg.in_h;
    gemms.reserve(static_cast<size_t>(cfg.num_block) * 15 + 10);
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
          if (int e = add(d, pre + "conv" + std::to_string(k + 1) + " " + std::to_string(nf + gc * k) + "->32 lrelu"))
            return e;
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
        if (int e = add(d, pre + "conv5 192->64" + (r < 2 ? " x0.2 + x" : " x0.04 + 0.2 r + x_rrdb"))) return e;
      }
      cur = nxt;
    }
    {
      GemmDesc d = desc(X[cur], nf, cat, W, H, body_conv.w, nf, body_conv.b, t, nf, 0);
      d.resid = X[0];
      d.ldr = cat;
      if (int e = add(d, "conv_body + feat")) return e;
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
        if (int e = add(d, std::string("conv_up") + char('1' + s) + " parity " + char('0' + py) + char('0' + px) + " lrelu"))
          return e;
      }
    GemmDesc d = desc(u2, nf, nf, 4 * W, 4 * H, hr.w, nf, hr.b, h, nf, 2);
    return add(d, "conv_hr lrelu");
  }
};

int run_gemms(EsrEngine* E, cudaStream_t st) {
  for (const GemmLaunch& L : E->gemms)
    if (int rc = launch_gemm(L, st)) return rc;
  return 0;
}

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
  E->dry = true;
  E->layout();
  E->cap = E->used;
  *out = reinterpret_cast<sdw_upsampler*>(E);
  return 0;
}

void sdw_upsampler_destroy(sdw_upsampler* e) {
  EsrEngine* E = reinterpret_cast<EsrEngine*>(e);
  if (E && E->graph_exec) cudaGraphExecDestroy(E->graph_exec);
  delete E;
}

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
  if (E->graph_exec) {
    cudaGraphExecDestroy(E->graph_exec);
    E->graph_exec = nullptr;
  }
  E->base = static_cast<uint8_t*>(arena);
  E->dry = false;
  E->layout();
  return E->build_ops();
}

int sdw_upsampler_num_params(const sdw_upsampler* e) {
  const EsrEngine* E = reinterpret_cast<const EsrEngine*>(e);
  return E ? static_cast<int>(E->order.size()) : 0;
}

int sdw_upsampler_param_info(const sdw_upsampler* e, int index, const char** name, int64_t* numel) {
  const EsrEngine* E = reinterpret_cast<const EsrEngine*>(e);
  SDW_REQUIRE(E && index >= 0 && index < static_cast<int>(E->order.size()), "bad index");
  if (name) *name = E->order[index].c_str();
  if (numel) *numel = E->params.at(E->order[index]).numel;
  return 0;
}

int sdw_upsampler_load_param(sdw_upsampler* e, const char* name, const void* src_f16, int64_t numel, void* stream) {
  EsrEngine* E = reinterpret_cast<EsrEngine*>(e);
  SDW_REQUIRE(E && name && src_f16 && !E->dry, "null / engine not bound");
  auto it = E->params.find(name);
  SDW_REQUIRE(it != E->params.end(), "unknown upsampler parameter");
  EsrParam& p = it->second;
  SDW_REQUIRE(numel == p.numel, "upsampler parameter size mismatch");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (p.kind == K_BIAS) {
    esr_bias_kernel<<<static_cast<unsigned>((numel + 255) / 256), 256, 0, st>>>(static_cast<const __half*>(src_f16),
                                                                               static_cast<float*>(p.dst),
                                                                               static_cast<int>(numel), p.scale);
    SDW_CUDA_OK(cudaGetLastError());
  } else if (p.kind == K_CONV3) {
    if (int rc = pack_weight(src_f16, p.N, p.C, 3, 3, 0, p.dst, st)) return rc;
  } else if (p.kind == K_UP4) {
    if (int rc = pack_weight_up4(src_f16, p.N, p.C, p.dst, st)) return rc;
  } else {
    SDW_CUDA_OK(cudaMemcpyAsync(p.dst, src_f16, static_cast<size_t>(numel) * 2, cudaMemcpyDeviceToDevice, st));
  }
  p.loaded = true;
  return 0;
}

int sdw_upsampler_missing_params(const sdw_upsampler* e, const char** first_missing) {
  const EsrEngine* E = reinterpret_cast<const EsrEngine*>(e);
  if (!E) return -1;
  int n = 0;
  for (auto& name : E->order)
    if (!E->params.at(name).loaded) {
      if (n == 0 && first_missing) *first_missing = name.c_str();
      ++n;
    }
  return n;
}

int sdw_upsampler_run(sdw_upsampler* e, const uint8_t* in_u8, uint8_t* out_u8, float* out_preclamp_f32, int use_graph,
                      void* stream) {
  EsrEngine* E = reinterpret_cast<EsrEngine*>(e);
  SDW_REQUIRE(E && in_u8 && out_u8 && !E->dry, "null / engine not bound");
  SDW_REQUIRE(sdw_upsampler_missing_params(e, nullptr) == 0, "upsampler parameters not loaded");
  const sdw_upsampler_config& c = E->cfg;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDW_REQUIRE(!use_graph || st != nullptr, "graph capture needs a real stream, not the legacy default stream 0");
  // the edge convs read / write the caller's buffers directly; the GEMM sequence in between works on the arena only and
  // is what the CUDA graph holds
  if (int rc = conv_first_u8(in_u8, c.frames, c.in_h, c.in_w, E->first.w, E->first.b, c.num_feat, E->X[0],
                             c.num_feat + 4 * c.num_grow_ch, st))
    return rc;
  if (use_graph) {
    if (!E->graph_exec) {
      cudaGraph_t graph = nullptr;
      SDW_CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      int rc = run_gemms(E, st);
      cudaError_t ce = cudaStreamEndCapture(st, &graph);
      if (rc) {
        if (graph) cudaGraphDestroy(graph);
        return rc;
      }
      SDW_CUDA_OK(ce);
      SDW_CUDA_OK(cudaGraphInstantiate(&E->graph_exec, graph, 0));
      cudaGraphDestroy(graph);
    }
    SDW_CUDA_OK(cudaGraphLaunch(E->graph_exec, st));
  } else {
    if (int rc = run_gemms(E, st)) return rc;
  }
  return conv_out_small(E->h, c.num_feat, c.frames, 4 * c.in_h, 4 * c.in_w, c.num_feat, E->last.w, E->last.b, 3,
                        out_preclamp_f32, out_u8, st, 1);
}

// tooling: CUDA-event time of every op of one forward after one untimed pass, written as "upsampler<TAB>index<TAB>
// microseconds<TAB>tag" lines.  The edge convs read / write dead arena regions here (their values do not matter).
int sdw_upsampler_debug_profile(sdw_upsampler* e, const char* path, void* stream) {
  EsrEngine* E = reinterpret_cast<EsrEngine*>(e);
  SDW_REQUIRE(E && path && !E->dry, "engine not bound");
  SDW_REQUIRE(sdw_upsampler_missing_params(e, nullptr) == 0, "upsampler parameters not loaded");
  const sdw_upsampler_config& c = E->cfg;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<std::function<int()>> ops;
  std::vector<std::string> tags;
  const uint8_t* in_scratch = E->Q;  // dead while conv_first runs
  uint8_t* out_scratch = E->P;       // dead while conv_last runs
  ops.push_back([=] {
    return conv_first_u8(in_scratch, c.frames, c.in_h, c.in_w, E->first.w, E->first.b, c.num_feat, E->X[0],
                         c.num_feat + 4 * c.num_grow_ch, st);
  });
  tags.push_back("conv_first u8 3->64 (CUDA cores)");
  for (size_t i = 0; i < E->gemms.size(); ++i) {
    ops.push_back([=] { return launch_gemm(E->gemms[i], st); });
    tags.push_back(E->tags[i]);
  }
  ops.push_back([=] {
    return conv_out_small(E->h, c.num_feat, c.frames, 4 * c.in_h, 4 * c.in_w, c.num_feat, E->last.w, E->last.b, 3,
                          nullptr, out_scratch, st, 1);
  });
  tags.push_back("conv_last 64->3 + uint8 (CUDA cores)");
  for (auto& op : ops)
    if (int rc = op()) return rc;
  FILE* f = std::fopen(path, "w");
  SDW_REQUIRE(f, "cannot open the profile file");
  const size_t n = ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& x : ev) cudaEventCreate(&x);
  int rc = 0;
  cudaEventRecord(ev[0], st);
  for (size_t i = 0; i < n && !rc; ++i) {
    rc = ops[i]();
    cudaEventRecord(ev[i + 1], st);
  }
  cudaStreamSynchronize(st);
  for (size_t i = 0; i < n && !rc; ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
    std::fprintf(f, "upsampler\t%zu\t%.2f\t%s\n", i, ms * 1e3f, tags[i].c_str());
  }
  for (auto& x : ev) cudaEventDestroy(x);
  std::fclose(f);
  if (rc) return rc;
  SDW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
