// sdw_model.cu — host scaffolding shared by the four engines (sampler, CLIP text tower, upsampler, safety checker): the
// arena bump allocator, the parameter table and its load dispatch, op lists, CUDA-graph replay and the per-op profile.
#include "sdw_internal.h"

#include <algorithm>
#include <memory>

namespace sdw {

void* Arena::take(size_t bytes) {
  off = (off + align - 1) / align * align;
  void* p = base ? base + off : nullptr;
  off += bytes;
  peak = std::max(peak, off);
  return p;
}

// ---- parameters ------------------------------------------------------------------------------------
void ParamTable::clear(bool bound_arena) {
  bound = bound_arena;
  slots.clear();
  index.clear();
}

void ParamTable::add(const std::string& name, ParamKind kind, void* dst, int64_t numel, int N, int C, int kh, int kw,
                     int geglu, float scale) {
  Param p{name, kind, dst, numel, N, C, kh, kw, geglu, scale, false};
  auto it = index.find(name);
  if (it != index.end()) {
    slots[it->second] = p;
  } else {
    index.emplace(name, size());
    slots.push_back(p);
  }
}

int ParamTable::info(int i, const char** name, int64_t* numel) const {
  SDW_REQUIRE(i >= 0 && i < size(), "bad parameter index");
  if (name) *name = slots[i].name.c_str();
  if (numel) *numel = slots[i].numel;
  return 0;
}

Param* ParamTable::find(const std::string& name) {
  auto it = index.find(name);
  return it == index.end() ? nullptr : &slots[it->second];
}

int ParamTable::missing(const char** first) const {
  int n = 0;
  for (const Param& p : slots)
    if (!p.loaded) {
      if (n == 0 && first) *first = p.name.c_str();
      ++n;
    }
  return n;
}

int ParamTable::load(const char* name, const void* src_f16, int64_t numel, cudaStream_t st) {
  SDW_REQUIRE(name && src_f16, "null");
  if (!bound) {
    set_error(std::string("engine not bound to an arena: cannot load ") + name);
    return 1;
  }
  Param* p = find(name);
  if (!p) {
    set_error(std::string("unknown parameter: ") + name);
    return 1;
  }
  if (p->numel != numel) {
    set_error(std::string("parameter size mismatch for ") + name + ": expected " + std::to_string(p->numel) + ", got " +
              std::to_string(numel));
    return 1;
  }
  int rc = 0;
  switch (p->kind) {
    case PACKED: rc = pack_weight(src_f16, p->N, p->C, p->kh, p->kw, p->geglu, p->dst, st); break;
    case PACKED_UP4: rc = pack_weight_up4(src_f16, p->N, p->C, p->dst, st); break;
    case RAW:
      SDW_CUDA_OK(cudaMemcpyAsync(p->dst, src_f16, static_cast<size_t>(numel) * 2, cudaMemcpyDeviceToDevice, st));
      break;
    case VEC:
      rc = half_to_float(static_cast<const __half*>(src_f16), static_cast<float*>(p->dst), numel, p->geglu ? p->N : 0,
                         p->scale, st);
      break;
  }
  if (rc == 0) p->loaded = true;
  return rc;
}

// ---- op lists, graphs, profiles --------------------------------------------------------------------
int OpList::run(cudaStream_t st, int step) const {
  for (const OpFn& f : ops)
    if (int rc = f(st, step)) return rc;
  return 0;
}

void OpList::add(const std::string& tag, OpFn f) {
  ops.push_back(std::move(f));
  tags.push_back(tag);
  launches += 1;
}

int OpList::add_gemm(const GemmDesc& d, const std::string& tag) {
  auto L = std::make_shared<GemmLaunch>();
  if (int e = plan_gemm(d, L.get())) {
    set_error(tag + ": " + last_error());
    return e;
  }
  add(tag, [L](cudaStream_t st, int) { return launch_gemm(*L, st); });
  return 0;
}

void OpList::append(const OpList& o) {
  ops.insert(ops.end(), o.ops.begin(), o.ops.end());
  tags.insert(tags.end(), o.tags.begin(), o.tags.end());
  launches += o.launches;
}

void GraphCache::reset() {
  if (exec) cudaGraphExecDestroy(exec);
  exec = nullptr;
}

int GraphCache::launch(int k, cudaStream_t st, const std::function<int(cudaStream_t)>& body) {
  if (!exec || key != k) {
    reset();
    cudaGraph_t graph = nullptr;
    SDW_CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    int rc = body(st);
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    SDW_CUDA_OK(ce);
    SDW_CUDA_OK(cudaGraphInstantiate(&exec, graph, 0));
    cudaGraphDestroy(graph);
    key = k;
  }
  SDW_CUDA_OK(cudaGraphLaunch(exec, st));
  return 0;
}

int profile_ops(FILE* f, const char* section, const OpList& ops, cudaStream_t st, int step) {
  if (int rc = ops.run(st, step)) return rc;
  const size_t n = ops.ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& x : ev) cudaEventCreate(&x);
  int rc = 0;
  cudaEventRecord(ev[0], st);
  for (size_t i = 0; i < n && !rc; ++i) {
    rc = ops.ops[i](st, step);
    cudaEventRecord(ev[i + 1], st);
  }
  cudaStreamSynchronize(st);
  for (size_t i = 0; i < n && !rc; ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
    std::fprintf(f, "%s\t%zu\t%.2f\t%s\n", section, i, ms * 1e3f, ops.tags[i].c_str());
  }
  for (auto& x : ev) cudaEventDestroy(x);
  return rc;
}

}  // namespace sdw
