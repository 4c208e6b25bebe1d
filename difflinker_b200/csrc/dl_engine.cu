// difflinker_b200 engine: C-ABI (include/difflinker_b200.h), weight packing, workspace, launch sequences,
// CUDA-graph replay of the reverse-diffusion loop. Kernels live in kernels_simt.cuh / kernels_tc.cuh.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <map>
#include <string>
#include <vector>

#include "../../include/difflinker_b200.h"
#include "kernels_simt.cuh"
#include "kernels_tc.cuh"
#include "kernels_node_tc.cuh"
#include "kernels_retry.cuh"

using namespace dl;

static thread_local char g_err[1024] = "";
static void set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t _e = (call);                                                              \
    if (_e != cudaSuccess) {                                                              \
      set_err("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e));       \
      return DL_ERR_CUDA;                                                                 \
    }                                                                                     \
  } while (0)

namespace {

struct Workspace {
  int B = 0, N = 0;
  float *nm = nullptr, *x0 = nullptr, *xa = nullptr, *xb = nullptr, *h = nullptr, *ABg = nullptr, *ABc = nullptr,
        *agg = nullptr, *z = nullptr, *ABgmax = nullptr, *ABcmax = nullptr, *eps = nullptr;
  int* cls = nullptr;
  // cut-off graphs on the tensor-core path: per-row neighbour lists and packed tile records of the current call (k_nbr)
  int *nbr = nullptr, *recs = nullptr, *xrecs = nullptr, *n_recs = nullptr;
  float4 *x04 = nullptr, *xa4 = nullptr, *xb4 = nullptr;
  int *rowidx = nullptr, *colidx = nullptr, *xrowidx = nullptr, *nr = nullptr, *nc = nullptr, *nxr = nullptr,
      *n_items = nullptr, *xmols = nullptr, *n_xmols = nullptr, *n_xitems = nullptr;
  int4* items = nullptr;
  int4* xitems = nullptr;
  int* tile_ctr = nullptr;
  unsigned long long* seeds = nullptr;   // dl_sample_chain_seeded: the call's B seeds, read by the captured step
  std::vector<void*> allocs;
};

struct HostStage {  // device staging for the *_host entry points, and the sub-batch rows of dl_sample_chain_retry
  size_t cap = 0;
  char* buf = nullptr;
};

// DL_TIME_KERNELS=1: CUDA-event time of every launch of a (non-captured) forward, accumulated per kernel label and printed
// when the engine is destroyed -- the live (warm-cache, back-to-back) counterpart of the ncu launch list. One record per
// engine, so engines driven from separate host threads (EDM.devices) share no state.
struct KernelTimes {
  bool on = false;
  struct Rec { const char* label; cudaEvent_t a, b; };
  std::vector<Rec> pending;
  std::map<std::string, std::pair<double, long>> acc;
  void begin(cudaStream_t st, const char* label) {
    if (!on) return;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    if (cap != cudaStreamCaptureStatusNone) return;
    Rec r{label, nullptr, nullptr};
    cudaEventCreate(&r.a); cudaEventCreate(&r.b);
    cudaEventRecord(r.a, st);
    pending.push_back(r);
  }
  void end(cudaStream_t st) {
    if (!on || pending.empty() || pending.back().b == nullptr) return;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    if (cap != cudaStreamCaptureStatusNone) return;
    cudaEventRecord(pending.back().b, st);
  }
  void collect(cudaStream_t st) {
    if (!on || pending.empty()) return;
    cudaStreamSynchronize(st);
    for (auto& r : pending) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { auto& a = acc[r.label]; a.first += ms; a.second += 1; }
      cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    }
    pending.clear();
  }
  void report() {
    if (!on || acc.empty()) return;
    double tot = 0;
    for (auto& kv : acc) tot += kv.second.first;
    for (auto& kv : acc)
      fprintf(stderr, "[dl times] %-22s %6ld launches  avg %8.2f us  share %5.1f%%\n", kv.first.c_str(), kv.second.second,
              1e3 * kv.second.first / kv.second.second, 100.0 * kv.second.first / tot);
  }
};

}  // namespace

struct dl_engine {
  dl_config cfg{};
  dl_egnn_options opts{};
  int D = 0;
  int num_sms = 0;
  int max_threads_per_sm = 2048;
  int slice_B_full = 0, slice_b0 = 0;   // dl_set_noise_slice: this engine samples rows [b0, b0 + B) of a B_full batch
  // dl_set_start_step: the linker sampler starts at step start_step from q(z_t0 | x) with these scalars; -1: from noise at T
  int start_step = -1;
  float start_alpha = 0.f, start_sigma = 0.f;
  // dl_set_start_steps: molecule b of the following calls starts at step starts_t0[b] with its own scalars; empty: none
  std::vector<int32_t> starts_t0;
  std::vector<float> starts_alpha, starts_sigma;
  HostStage start_rows;        // a per-molecule start-step call's row order, lags, scalars and gathered inputs
  // dl_set_resamplings: the inpainting sampler runs `resamplings` passes per reverse step, for calls of T = resample_T,
  // re-noising with the (T, 2) (alpha_t|s, sigma_t|s) of `jump`; 1: the plain loop. coef_passes: the device table's host copy.
  int resamplings = 1, resample_T = 0;
  std::vector<float> jump;
  std::vector<dl_step_coef> coef_passes;
  // dl_set_clash_guidance: the linker sampler pushes linker atoms out of the pocket at its last guide_steps reverse steps
  // with guide_scale, by the (guide_types, guide_types) table guide_table (pm); guide_steps = 0: off. Each sampling call
  // uploads the table to guide_clash (guide_cap floats) on its loop stream, as it uploads its coefficient table.
  float guide_scale = 0.f;
  int guide_steps = 0, guide_types = 0;
  std::vector<float> guide_table;
  float* guide_clash = nullptr;
  size_t guide_cap = 0;
  // dl_set_solver: the linker sampler's update for calls of T = solver_T, from the (solver_T + 1, 8) table solver_table
  // (host copy), which each call uploads after its coefficient rows; DL_SOLVER_ANCESTRAL: the plain loop
  int solver_kind = DL_SOLVER_ANCESTRAL, solver_T = 0;
  std::vector<float> solver_table;
  int64_t mol_steps = 0;      // dl_last_molecule_steps
  bool finalized = false;
  std::map<std::string, std::vector<float>> raw;
  float* wblob = nullptr;      // packed fp32 weights
  __half* wblob_tc = nullptr;  // packed fp16 hi/lo tiles
  std::vector<GclW> gcl;       // [L*S]
  std::vector<EqW> eq;         // [L]
  const float *We_t = nullptr, *be = nullptr, *Wo = nullptr, *bo = nullptr;
  Workspace ws;
  // dl_sample_chain_retry: the loop workspace of the failed molecules' sub-batch (cached by (B', N) like ws, which it
  // never frees or resizes), their gathered inputs and chain, and the events of the rounds (ev_r*: the sub-batch loop's
  // own, so ev_t0/ev_t1 keep timing the first loop; ev_g*: one round, gather to scatter)
  Workspace ws_sub;
  HostStage sub_rows;
  HostStage hashes;            // DL_CHECK_UNIQUE: the full batch's graph hashes, (B) uint64, grown to the largest B
  // dl_set_ring_sizes: the ring sizes DL_CHECK_RINGS allows (ring_set: set at least once). ring_masks: the ring-size masks
  // of the last dl_sample_chain_retry call's ring_B rows, grown to the largest B; ring_B = 0 when it did not require the bit
  bool ring_set = false;
  unsigned long long ring_allowed = 0;
  HostStage ring_masks;
  int ring_B = 0;
  // dl_set_anchors: the (anchors_B, anchors_N) int8 anchor flags of the next dl_sample_chain_retry call, which clears
  // anchors_set; the buffer is kept, grown to the largest B * N
  HostStage anchors;
  bool anchors_set = false;
  int anchors_B = 0, anchors_N = 0;
  // dl_set_fixed_atoms: the (fixed_B, fixed_N) int8 flags of the linker rows the next dl_sample_chain* call keeps (in the
  // buffer, followed by two ints of the call's vetting) and the host copy of the (fixed_T + 1, 2) scalars; that call reads
  // and clears fixed_set, and its recovery rounds gather the flags of their rows
  HostStage fixed;
  bool fixed_set = false;
  int fixed_B = 0, fixed_N = 0, fixed_T = 0;
  std::vector<float> fixed_scalars;
  // dl_set_linker_types: host copies of the (types_B) masks of allowed type channels and the (types_T + 1, 2) scalars; the
  // next dl_sample_chain* call reads and clears types_set and uploads them, and its recovery rounds take their rows' masks
  bool types_set = false;
  int types_B = 0, types_T = 0;
  std::vector<uint32_t> types_masks;
  std::vector<float> types_scalars;
  cudaEvent_t ev_r0 = nullptr, ev_r1 = nullptr, ev_g0 = nullptr, ev_g1 = nullptr;
  float retry_ms = 0.f;
  cudaStream_t loop_stream = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
  float* coef_dev = nullptr;
  int coef_cap = 0;            // bytes of coef_dev
  int* step_ctr = nullptr;     // [3]: step_prep, step_fin, and with resampling the step k_finish tags NaN flags with
  int64_t launches = 0;
  HostStage stage;
  KernelTimes times;           // DL_TIME_KERNELS
  bool use_tc = false;
  // pointers of the most recent forward (for dl_time_edge_kernel)
  const int8_t* last_edge_mask = nullptr;
  const float* last_linker_mask = nullptr;
  int last_B = 0, last_N = 0;
};

namespace {

// edge-attribute columns of every edge MLP's first layer: [d, d0], or their 24 sinusoidal features
int edges_in(const dl_engine* e) { return e->opts.sin_embedding ? N_SIN_FEAT : 2; }

#define TIMED(label, stream, stmt) do { e->times.begin(stream, label); stmt; e->times.end(stream); } while (0)

struct ExpectedParam {
  std::string name;
  int64_t numel;
};

// edges_in: width of the edge attributes of every edge MLP's first layer (2 distances, or 24 with sin_embedding)
std::vector<ExpectedParam> expected_params(const dl_config& c, int edges_in) {
  const int D = c.in_node_nf + c.context_node_nf + (c.condition_time ? 1 : 0);
  const int Hh = c.hidden_nf;
  std::vector<ExpectedParam> v;
  v.push_back({"dynamics.embedding.weight", (int64_t)Hh * D});
  v.push_back({"dynamics.embedding.bias", Hh});
  v.push_back({"dynamics.embedding_out.weight", (int64_t)D * Hh});
  v.push_back({"dynamics.embedding_out.bias", D});
  char buf[160];
  for (int l = 0; l < c.n_layers; ++l) {
    for (int s = 0; s < c.inv_sublayers; ++s) {
      snprintf(buf, sizeof(buf), "dynamics.e_block_%d.gcl_%d.", l, s);
      std::string p(buf);
      v.push_back({p + "edge_mlp.0.weight", (int64_t)Hh * (2 * Hh + edges_in)});
      v.push_back({p + "edge_mlp.0.bias", Hh});
      v.push_back({p + "edge_mlp.2.weight", (int64_t)Hh * Hh});
      v.push_back({p + "edge_mlp.2.bias", Hh});
      v.push_back({p + "node_mlp.0.weight", (int64_t)Hh * 2 * Hh});
      v.push_back({p + "node_mlp.0.bias", Hh});
      v.push_back({p + "node_mlp.2.weight", (int64_t)Hh * Hh});
      v.push_back({p + "node_mlp.2.bias", Hh});
    }
    snprintf(buf, sizeof(buf), "dynamics.e_block_%d.gcl_equiv.", l);
    std::string p(buf);
    v.push_back({p + "coord_mlp.0.weight", (int64_t)Hh * (2 * Hh + edges_in)});
    v.push_back({p + "coord_mlp.0.bias", Hh});
    v.push_back({p + "coord_mlp.2.weight", (int64_t)Hh * Hh});
    v.push_back({p + "coord_mlp.2.bias", Hh});
    v.push_back({p + "coord_mlp.4.weight", Hh});
  }
  return v;
}

using RawWeights = std::map<std::string, std::vector<float>>;

// Host-side packer: appends 16-byte aligned fp32 segments to one blob and fp16 tensor-core tiles to another, and remembers
// which weight-record field each belongs to; point() aims those fields at the uploaded blobs.
struct Packer {
  std::vector<float> blob;
  std::vector<__half> tc;
  std::vector<std::pair<const float**, size_t>> fields;
  std::vector<std::pair<const void**, size_t>> tc_fields;
  void add(const float** field, const std::vector<float>& seg) {
    while (blob.size() % 4) blob.push_back(0.f);
    fields.push_back({field, blob.size()});
    blob.insert(blob.end(), seg.begin(), seg.end());
  }
  void add_tc(const void** field, size_t off) { tc_fields.push_back({field, off}); }
  void point(const float* base, const __half* tc_base) const {
    for (auto& f : fields) *f.first = base + f.second;
    for (auto& f : tc_fields) *f.first = tc_base + f.second;
  }
};

// (out,in) row-major sub-block [0:out) x [c0:c0+k) -> k-major [k][out]
std::vector<float> transpose_block(const std::vector<float>& W, int out, int in_stride, int c0, int k) {
  std::vector<float> t((size_t)k * out);
  for (int o = 0; o < out; ++o)
    for (int i = 0; i < k; ++i) t[(size_t)i * out + o] = W[(size_t)o * in_stride + c0 + i];
  return t;
}
std::vector<float> column(const std::vector<float>& W, int out, int in_stride, int c) {
  std::vector<float> t(out);
  for (int o = 0; o < out; ++o) t[o] = W[(size_t)o * in_stride + c];
  return t;
}

// fp32 k-major copies of an edge MLP (prefix p: "...edge_mlp." or "...coord_mlp.") whose first Linear reads in1 inputs:
// everything but the input-distance column w0, which only the denoiser has.
void pack_edge_mlp(Packer& pk, EdgeMlpW& w, const RawWeights& raw, const std::string& p, int in1) {
  const auto& W1 = raw.at(p + "0.weight");
  pk.add(&w.W1a_t, transpose_block(W1, H, in1, 0, H));
  pk.add(&w.W1b_t, transpose_block(W1, H, in1, H, H));
  pk.add(&w.b1, raw.at(p + "0.bias"));
  pk.add(&w.wd, column(W1, H, in1, 2 * H));
  pk.add(&w.W2_t, transpose_block(raw.at(p + "2.weight"), H, H, 0, H));
  pk.add(&w.b2, raw.at(p + "2.bias"));
}

// fp32 k-major copies of a GCL (prefix p ends in '.'): its edge MLP and its node MLP.
void pack_gcl(Packer& pk, GclW& w, const RawWeights& raw, const std::string& p, int in1) {
  pack_edge_mlp(pk, w, raw, p + "edge_mlp.", in1);
  pk.add(&w.W3_t, transpose_block(raw.at(p + "node_mlp.0.weight"), H, 2 * H, 0, 2 * H));
  pk.add(&w.b3, raw.at(p + "node_mlp.0.bias"));
  pk.add(&w.W4_t, transpose_block(raw.at(p + "node_mlp.2.weight"), H, H, 0, H));
  pk.add(&w.b4, raw.at(p + "node_mlp.2.bias"));
}

// The denoiser's additions to an edge MLP (first Linear over IN1 = 2H+2 inputs, or 2H+24 with sin_embedding): the
// input-distance column w0 (or the 24 embedding columns), the bounds of the edge-attribute columns, and the tensor-core
// copies -- W2 and the log2-domain first layer (kernels_tc.cuh pack_w2).
void pack_edge_mlp_denoiser(Packer& pk, EdgeMlpW& w, const RawWeights& raw, const std::string& p, bool sin_embedding) {
  const int IN1 = 2 * H + (sin_embedding ? N_SIN_FEAT : 2);
  auto scaled = [](const std::vector<float>& v) { std::vector<float> o(v.size()); for (size_t i = 0; i < v.size(); ++i) o[i] = (float)((double)v[i] * tc::NEG_LOG2E); return o; };
  auto absmax = [](const std::vector<float>& v) { float m = 0.f; for (float x : v) m = std::max(m, std::fabs(x)); return m; };
  const auto& W1 = raw.at(p + "0.weight");
  const std::vector<float> wd = column(W1, H, IN1, 2 * H), w0 = column(W1, H, IN1, 2 * H + 1);
  pk.add(&w.w0, w0);
  pk.add_tc(&w.W2_tc, tc::pack_w2(raw.at(p + "2.weight"), pk.tc, &w.w2_descale));
  pk.add_tc(&w.W1_tc, tcn::pack_blocks(scaled(W1), IN1, 2, pk.tc, &w.w1_descale));
  pk.add(&w.b1_u, scaled(raw.at(p + "0.bias")));
  pk.add(&w.wd_u, scaled(wd));
  pk.add(&w.w0_u, scaled(w0));
  w.wdmax = absmax(wd); w.w0max = absmax(w0);
  if (sin_embedding) {
    const std::vector<float> we = transpose_block(W1, H, IN1, 2 * H, N_SIN_FEAT);
    pk.add(&w.we, we);
    pk.add(&w.we_u, scaled(we));
    w.wdmax = 0.f; w.w0max = 0.f;
    for (int k = 0; k < N_SIN_FEAT; ++k) w.wdmax += absmax(std::vector<float>(we.begin() + k * H, we.begin() + (k + 1) * H));
  }
}

template <typename T>
dl_status upload_blob(const std::vector<T>& host, T** dev) {
  if (*dev) cudaFree(*dev);
  *dev = nullptr;
  CK(cudaMalloc((void**)dev, std::max<size_t>(host.size(), 1) * sizeof(T)));
  CK(cudaMemcpy(*dev, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice));
  return DL_OK;
}

template <typename T>
dl_status dev_alloc(Workspace& ws, T** p, size_t count) {
  void* q = nullptr;
  CK(cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T)));
  ws.allocs.push_back(q);
  *p = reinterpret_cast<T*>(q);
  return DL_OK;
}

void free_workspace(Workspace& ws) {
  for (void* p : ws.allocs) cudaFree(p);
  ws = Workspace();
}

dl_status ensure_workspace(dl_engine* e, int B, int N) {
  Workspace& ws = e->ws;
  if (ws.B == B && ws.N == N) return DL_OK;
  free_workspace(ws);
  const size_t n = (size_t)B * N;
  const int xd = 3 + e->cfg.in_node_nf;
  dl_status s;
#define WSA(field, cnt) if ((s = dev_alloc(ws, &ws.field, (cnt))) != DL_OK) return s
  WSA(nm, n); WSA(x0, n * 3); WSA(xa, n * 3); WSA(xb, n * 3); WSA(h, n * H); WSA(ABg, n * 2 * H); WSA(ABc, n * 2 * H);
  WSA(agg, n * H); WSA(z, n * xd); WSA(eps, n * xd); WSA(cls, n); WSA(x04, n); WSA(xa4, n); WSA(xb4, n); WSA(ABgmax, n * 2); WSA(ABcmax, n * 2);
  WSA(rowidx, n); WSA(colidx, n); WSA(xrowidx, n); WSA(nr, B); WSA(nc, B); WSA(nxr, B); WSA(n_items, 1);
  WSA(xmols, B); WSA(n_xmols, 1); WSA(items, n); WSA(xitems, n); WSA(n_xitems, 1); WSA(tile_ctr, 64); WSA(seeds, B);
  if (e->use_tc && e->cfg.graph_type != 0) { WSA(nbr, n * N); WSA(recs, n * CUT_REC); WSA(xrecs, n * CUT_REC); WSA(n_recs, 2); }
#undef WSA
  ws.B = B; ws.N = N;
  return DL_OK;
}

Plan make_plan(const Workspace& ws) {
  Plan p;
  p.rowidx = ws.rowidx; p.colidx = ws.colidx; p.xrowidx = ws.xrowidx; p.nr = ws.nr; p.nc = ws.nc; p.nxr = ws.nxr;
  p.items = ws.items; p.n_items = ws.n_items; p.xmols = ws.xmols; p.n_xmols = ws.n_xmols;
  p.xitems = ws.xitems; p.n_xitems = ws.n_xitems;
  return p;
}

Geom make_geom(const dl_engine* e, int B, int N) {
  Geom g;
  g.B = B; g.N = N; g.F = e->cfg.in_node_nf; g.C = e->cfg.context_node_nf; g.D = e->D;
  g.graph_type = e->cfg.graph_type; g.norm_constant = e->cfg.norm_constant;
  g.normalization_factor = e->cfg.normalization_factor;
  return g;
}

#define LAUNCH_CHECK()                                                                    \
  do {                                                                                    \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess) {                                                              \
      set_err("%s:%d kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e));   \
      return DL_ERR_CUDA;                                                                 \
    }                                                                                     \
  } while (0)

// The work plan of ws (2 launches): live rows and columns of every molecule, then work items of at most tile_edges edges and
// max_rows rows. Masks are constant over a whole sample_chain: the plan is built once per call.
// k_plan_mol stages two ints per row in dynamic shared memory, which it gets without raising its attribute: N <= 6144.
constexpr int PLAN_MAX_N = 48 * 1024 / (2 * (int)sizeof(int));

dl_status build_plan(Workspace& ws, int B, int N, int graph_type, const int8_t* node_mask, const float* linker_mask,
                     const int8_t* edge_mask, int tile_edges, int max_rows, cudaStream_t st) {
  if (N > PLAN_MAX_N) {
    set_err("N = %d exceeds the work plan's limit of %d rows per molecule", N, PLAN_MAX_N);
    return DL_ERR_UNSUPPORTED;
  }
  CK(cudaMemsetAsync(ws.agg, 0, (size_t)B * N * H * sizeof(float), st));  // dead rows aggregate to exactly 0
  k_plan_mol<<<B, 256, 2 * N * sizeof(int), st>>>(N, graph_type, edge_mask, node_mask, linker_mask, ws.rowidx,
                                                  ws.colidx, ws.xrowidx, ws.nr, ws.nc, ws.nxr);
  LAUNCH_CHECK();
  k_plan_items<<<1, 1, 0, st>>>(B, tile_edges, max_rows, 1, max_rows, ws.nr, ws.nc, ws.nxr, ws.items, ws.n_items, ws.xmols,
                                ws.n_xmols, ws.xitems, ws.n_xitems);
  LAUNCH_CHECK();
  return DL_OK;
}

// The denoiser's plan, tiled for the edge kernel it runs.
dl_status build_forward_plan(dl_engine* e, int B, int N, const int8_t* node_mask, const float* linker_mask,
                             const int8_t* edge_mask, cudaStream_t st) {
  const dl_status s = build_plan(e->ws, B, N, e->cfg.graph_type, node_mask, linker_mask, edge_mask,
                                 e->use_tc ? tc::TN : ET, e->use_tc ? tc::MAXR : MAXR, st);
  if (s == DL_OK) e->launches += 2;
  return s;
}

struct FwdIO {
  // Dynamics.forward mode
  const float* xh = nullptr; const float* t = nullptr; int t_numel = 0; float* out = nullptr;
  // common
  const int8_t* node_mask = nullptr; const float* linker_mask = nullptr; const int8_t* edge_mask = nullptr;
  const float* context = nullptr; int* nan_flags = nullptr;
  // sampler mode
  bool sampler = false; bool inpaint = false; const float* xh0 = nullptr; const float* upd_linker_mask = nullptr;
  const float* fragment_mask = nullptr; const float* noise = nullptr; float* chain = nullptr;
  NoiseRng rng{};
  int T = 0; float norm0 = 1.f, norm1 = 1.f, bias1 = 0.f;
  RowStarts rows{};   // per-molecule start steps, or rows.lag = null
  int R = 1; const float* jump = nullptr;   // resampling passes per reverse step (dl_set_resamplings), T counting passes
  const float* ode = nullptr;               // the solver rows of the loop (dl_set_solver), or null: the ancestral update
  const int8_t* fixed = nullptr;            // fixed atoms (dl_set_fixed_atoms): the rows' flags, or null
  const float* fix = nullptr;               // ... and the (alpha_s, sigma_s) rows of the loop
  const uint32_t* types = nullptr;          // linker types (dl_set_linker_types): the molecules' masks, or null
  const float* tsc = nullptr;               // ... and the (alpha_t, sigma_t) rows of the loop
};

// The k_finish instantiation of a sampler step: per-molecule streams, an ODE solver, fixed atoms, linker types.
template <bool FIX, bool TYPES>
void (*finish_kernel(bool per_mol, bool ode))(Geom, FinishArgs) {
  return ode ? (per_mol ? k_finish<true, true, FIX, TYPES> : k_finish<false, true, FIX, TYPES>)
             : (per_mol ? k_finish<true, false, FIX, TYPES> : k_finish<false, false, FIX, TYPES>);
}

ProjW proj_of(const EdgeMlpW& w) { return ProjW{w.W1a_t, w.W1b_t, w.b1}; }

// Arguments of one edge-kernel launch over the coordinates x / x4: a GCL's edge MLP, which aggregates into ws.agg, or
// (coord) a coordinate MLP, which writes x_out / x4_out.
EdgeArgs edge_args(const dl_engine* e, const EdgeMlpW& w, bool coord, const int8_t* edge_mask, const float* linker_mask,
                   const float* x, const float4* x4, float* x_out = nullptr, float4* x4_out = nullptr,
                   const float* w5 = nullptr) {
  const Workspace& ws = e->ws;
  const float ksc = e->use_tc ? 1.4426950408889634f : 1.0f;   // log2-domain first layer on the tensor-core path
  EdgeArgs ea{};
  ea.AB = coord ? ws.ABc : ws.ABg; ea.ABmax = coord ? ws.ABcmax : ws.ABgmax;
  ea.w2_descale = w.w2_descale; ea.wdmax = w.wdmax * ksc; ea.w0max = w.w0max * ksc;
  ea.x = x; ea.x0 = ws.x0; ea.x4 = x4; ea.x04 = ws.x04; ea.x4_out = x4_out;
  ea.edge_mask = edge_mask; ea.cls = ws.cls; ea.nm = ws.nm; ea.linker_mask = linker_mask;
  ea.W2_t = w.W2_t; ea.b2 = w.b2; ea.wd = e->use_tc ? w.wd_u : w.wd; ea.w0 = e->use_tc ? w.w0_u : w.w0; ea.w5 = w5;
  ea.plan = make_plan(ws); ea.agg = coord ? nullptr : ws.agg; ea.x_out = x_out; ea.nbr = ws.nbr;
  ea.recs = coord ? ws.xrecs : ws.recs;
  ea.n_recs = coord && ws.n_recs ? ws.n_recs + 1 : ws.n_recs;
  ea.coords_range = e->opts.coords_range;
  ea.we = e->use_tc ? w.we_u : w.we;
  return ea;
}

// The edge-kernel OPT bits (common.cuh) of the engine's EGNN options; tanh only concerns the coordinate update.
int edge_opt(const dl_engine* e, bool coord) {
  return (coord && e->opts.tanh ? OPT_TANH : 0) | (e->opts.aggregation == DL_AGGR_MEAN ? OPT_MEAN : 0) |
         (e->opts.sin_embedding ? OPT_SIN : 0);
}

// The edge MLPs whose first-layer projections are taken from the h that GCL s of block l writes, with the AB / ABmax
// buffers they go to: the next GCL; after a block's last GCL, the block's coordinate MLP and the next block's GCL 0.
// s = -1 stands for the embedding, consumed by GCL 0 of block 0. Returns the count (1 or 2).
struct NodeConsumer { const EdgeMlpW* w; float* AB; float* ABmax; };
int node_consumers(const dl_engine* e, int l, int s, NodeConsumer c[2]) {
  const int L = e->cfg.n_layers, S = e->cfg.inv_sublayers;
  const Workspace& ws = e->ws;
  if (s + 1 < S) { c[0] = {&e->gcl[l * S + s + 1], ws.ABg, ws.ABgmax}; return 1; }
  c[0] = {&e->eq[l], ws.ABc, ws.ABcmax};
  if (l + 1 == L) return 1;
  c[1] = {&e->gcl[(l + 1) * S], ws.ABg, ws.ABgmax};
  return 2;
}

// The tensor-core node kernel after GCL s of block l (weights w): its node MLP, then the projections of the new h for the
// consumers. s = -1 skips the node MLP and only projects the embedded h for GCL 0 (w = that GCL).
tcn::NodeTcArgs node_tc_args(const dl_engine* e, const GclW& w, int l, int s) {
  const Workspace& ws = e->ws;
  tcn::NodeTcArgs ta{};
  ta.h = ws.h; ta.agg = ws.agg; ta.nm = ws.nm; ta.proj_only = s < 0;
  ta.w3 = reinterpret_cast<const __half*>(w.W3_tc); ta.w4 = reinterpret_cast<const __half*>(w.W4_tc);
  ta.b3 = w.b3; ta.b4 = w.b4; ta.w3_descale = w.w3_descale; ta.w4_descale = w.w4_descale;
  NodeConsumer c[2];
  ta.n_proj = node_consumers(e, l, s, c);
  for (int i = 0; i < ta.n_proj; ++i) {
    ta.pw[i] = reinterpret_cast<const __half*>(c[i].w->W1_tc); ta.pb1[i] = c[i].w->b1_u;
    ta.p_descale[i] = c[i].w->w1_descale; ta.AB[i] = c[i].AB; ta.ABmax[i] = c[i].ABmax;
  }
  ta.tile_nodes = tcn::pick_tile_nodes(ws.B * ws.N, e->num_sms);
  return ta;
}

// Every OPT combination of the SIMT edge kernel (tanh only for the coordinate update), walked at compile time.
template <bool COORD, int OPT = 0>
void launch_edge_simt(int opt, int num_sms, const Geom& gm, const EdgeArgs& ea, cudaStream_t st) {
  if constexpr (OPT <= (OPT_TANH | OPT_MEAN | OPT_SIN)) {
    if constexpr (COORD || !(OPT & OPT_TANH))
      if (opt == OPT) { k_edge_simt<COORD, ACT_SILU, OPT><<<num_sms, 256, EDGE_SIMT_SMEM, st>>>(gm, ea); return; }
    launch_edge_simt<COORD, OPT + 1>(opt, num_sms, gm, ea, st);
  }
}

template <bool COORD, int OPT = 0>
cudaError_t opt_in_edge_simt() {
  if constexpr (OPT > (OPT_TANH | OPT_MEAN | OPT_SIN)) {
    return cudaSuccess;
  } else {
    if constexpr (COORD || !(OPT & OPT_TANH)) {
      const cudaError_t err = cudaFuncSetAttribute(k_edge_simt<COORD, ACT_SILU, OPT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)EDGE_SIMT_SMEM);
      if (err != cudaSuccess) return err;
    }
    return opt_in_edge_simt<COORD, OPT + 1>();
  }
}

dl_status launch_edge(dl_engine* e, const Geom& gm, const EdgeArgs& ea, bool coord, const void* w2_tc, cudaStream_t st) {
  const int opt = edge_opt(e, coord);
  if (e->use_tc) {
    dl_status s = tc::launch_edge_tc(gm, ea, coord, opt, w2_tc, e->num_sms, st);
    if (s != DL_OK) { set_err("no tensor-core edge kernel for graph type %d with options %d", gm.graph_type, opt); return s; }
  } else if (coord) {
    launch_edge_simt<true>(opt, e->num_sms, gm, ea, st);
  } else {
    launch_edge_simt<false>(opt, e->num_sms, gm, ea, st);
  }
  LAUNCH_CHECK();
  e->launches += 1;
  return DL_OK;
}

// One Dynamics.forward worth of launches (1 + L*(2S+2) + 1 kernels).
dl_status enqueue_forward(dl_engine* e, int B, int N, const FwdIO& io, cudaStream_t st) {
  Workspace& ws = e->ws;
  const Geom gm = make_geom(e, B, N);
  const int n = B * N;
  const int L = e->cfg.n_layers, S = e->cfg.inv_sublayers;
  const int node_blocks = (n + NODE_TM - 1) / NODE_TM;
  const size_t node_smem = 3 * NODE_TM * LDX * sizeof(float);

  PrepArgs pa{};
  pa.xh = io.sampler ? ws.z : io.xh;
  pa.node_mask = io.node_mask; pa.linker_mask = io.linker_mask;
  pa.t = io.t; pa.t_numel = io.t_numel; pa.context = io.context;
  pa.We_t = e->We_t; pa.be = e->be; pa.proj = proj_of(e->gcl[0]);
  pa.nm = ws.nm; pa.x0 = ws.x0; pa.x = ws.xa; pa.x04 = e->use_tc ? ws.x04 : nullptr; pa.x4 = e->use_tc ? ws.xa4 : nullptr; pa.cls = ws.cls; pa.h = ws.h;
  pa.AB = e->use_tc ? nullptr : ws.ABg; pa.ABmax = ws.ABgmax;
  pa.coef = io.sampler ? e->coef_dev : nullptr;
  pa.step_prep = io.sampler ? e->step_ctr : nullptr;
  pa.step_fin = io.sampler ? e->step_ctr + 1 : nullptr;
  TIMED("k_prep", st, (launch_chain(k_prep, dim3(node_blocks), dim3(256), 0, st, gm, pa)));
  LAUNCH_CHECK();
  e->launches += 1;
  if (e->use_tc) {
    // A | B projections of block 0 / gcl 0 from the embedded h, on the tensor cores
    const tcn::NodeTcArgs ta = node_tc_args(e, e->gcl[0], 0, -1);
    TIMED("k_node_tc(proj only)", st, (tcn::launch_node(n, ta, st)));
    LAUNCH_CHECK();
    e->launches += 1;
  }

  if (ws.nbr != nullptr) {
    // the cut-off graph of this call (a function of its input coordinates): neighbour lists + packed tiles
    CK(cudaMemsetAsync(ws.n_recs, 0, 2 * sizeof(int), st));
    k_nbr<<<B, 512, (size_t)N * CUT_SMEM_PER_NODE, st>>>(N, e->cfg.graph_type, ws.x04, ws.cls, ws.rowidx, ws.colidx,
                                                        ws.xrowidx, ws.nr, ws.nc, ws.nxr, ws.nbr, ws.recs, ws.xrecs,
                                                        ws.n_recs);
    LAUNCH_CHECK();
    e->launches += 1;
  }

  float* xin = ws.xa;
  float* xout = ws.xb;
  float4* xin4 = ws.xa4;
  float4* xout4 = ws.xb4;
  e->last_edge_mask = io.edge_mask; e->last_linker_mask = io.linker_mask; e->last_B = B; e->last_N = N;
  for (int l = 0; l < L; ++l) {
    for (int s = 0; s < S; ++s) {
      const GclW& w = e->gcl[l * S + s];
      const EdgeArgs ea = edge_args(e, w, false, io.edge_mask, io.linker_mask, xin, xin4);
      e->times.begin(st, "edge GCL");
      dl_status st2 = launch_edge(e, gm, ea, false, w.W2_tc, st);
      e->times.end(st);
      if (st2 != DL_OK) return st2;

      if (e->use_tc) {
        const tcn::NodeTcArgs ta = node_tc_args(e, w, l, s);
        TIMED(ta.n_proj == 2 ? "k_node_tc(2 proj)" : "k_node_tc(1 proj)", st, (tcn::launch_node(n, ta, st)));
      } else {
        NodeArgs na{};
        na.h = ws.h; na.agg = ws.agg; na.nm = ws.nm; na.W3_t = w.W3_t; na.b3 = w.b3; na.W4_t = w.W4_t; na.b4 = w.b4;
        NodeConsumer c[2];
        const int n_proj = node_consumers(e, l, s, c);
        na.proj1 = proj_of(*c[0].w); na.AB1 = c[0].AB; na.ABmax1 = c[0].ABmax;
        if (n_proj == 2) { na.proj2 = proj_of(*c[1].w); na.AB2 = c[1].AB; na.ABmax2 = c[1].ABmax; }
        k_node<ACT_SILU><<<node_blocks, 256, node_smem, st>>>(n, na);
      }
      LAUNCH_CHECK();
      e->launches += 1;
    }
    k_copy_x<<<(n * 3 + 255) / 256, 256, 0, st>>>(n * 3, xin, xout, e->use_tc ? xin4 : nullptr, xout4);
    LAUNCH_CHECK();
    e->launches += 1;
    const EqW& w = e->eq[l];
    const EdgeArgs ea = edge_args(e, w, true, io.edge_mask, io.linker_mask, xin, xin4, xout, xout4, w.w5);
    e->times.begin(st, "edge COORD");
    dl_status st2 = launch_edge(e, gm, ea, true, w.W2_tc, st);
    e->times.end(st);
    if (st2 != DL_OK) return st2;
    std::swap(xin, xout);
    std::swap(xin4, xout4);
  }

  FinishArgs fa{};
  fa.h = ws.h; fa.x = xin; fa.x0 = ws.x0; fa.nm = ws.nm; fa.Wo = e->Wo; fa.bo = e->bo;
  fa.nan_flags = io.nan_flags;
  const bool fused_update = io.sampler && !io.inpaint;
  fa.out = fused_update ? nullptr : (io.sampler ? ws.eps : io.out);
  if (fused_update) {
    fa.z = ws.z; fa.fragment_mask = io.fragment_mask; fa.linker_mask = io.linker_mask; fa.noise = io.noise; fa.rng = io.rng;
    fa.coef = e->coef_dev; fa.step_fin = e->step_ctr + 1; fa.step_prep = e->step_ctr; fa.T = io.T;
    fa.norm0 = io.norm0; fa.norm1 = io.norm1; fa.bias1 = io.bias1; fa.chain = io.chain; fa.rows = io.rows;
    // the 2M history lives in ws.eps, which the fused linker update never writes otherwise
    fa.ode = io.ode; fa.hist = io.ode && e->solver_kind == DL_SOLVER_DPMPP_2M ? ws.eps : nullptr;
    fa.fixed = io.fixed; fa.xh0 = io.xh0; fa.fix = io.fix;
    fa.types = io.types; fa.tsc = io.tsc;
  } else if (io.sampler) {
    fa.tag_step = e->step_ctr + (io.R > 1 ? 2 : 1);   // with resampling the pass counter is not the step
  }
  const bool per_mol = io.rng.on == NOISE_PER_MOLECULE;
  auto* finish = fa.types ? (fa.fixed ? finish_kernel<true, true>(per_mol, fa.ode) : finish_kernel<false, true>(per_mol, fa.ode))
                          : (fa.fixed ? finish_kernel<true, false>(per_mol, fa.ode) : finish_kernel<false, false>(per_mol, fa.ode));
  TIMED("k_finish", st, (launch_chain(finish, dim3((n + 15) / 16), dim3(256), 0, st, gm, fa)));
  LAUNCH_CHECK();
  e->launches += 1;
  if (fused_update && e->guide_steps > 0) {
    // clash guidance (dl_set_clash_guidance): the step's z_s moved before anything reads it; the kernel returns at the
    // steps it does not guide, so one graph serves every step
    GuideArgs ga{};
    ga.xh = ws.z; ga.N = N; ga.row_stride = 3 + e->cfg.in_node_nf; ga.n_types = e->guide_types; ga.C = e->cfg.context_node_nf;
    ga.scale = e->guide_scale; ga.clash = e->guide_clash;
    ga.node_mask = io.node_mask; ga.linker_mask = io.linker_mask; ga.context = io.context;
    ga.step = e->step_ctr + 1; ga.T = io.T; ga.steps = e->guide_steps; ga.coef = e->coef_dev;
    ga.chain = io.chain; ga.norm0 = io.norm0; ga.fixed = io.fixed;
    TIMED("k_clash_guide", st, (launch_clash_guide(ga, B, st)));
    LAUNCH_CHECK();
    e->launches += 1;
  }
  if (e->cfg.centering || io.inpaint) {
    // per-molecule stage of inpainting models: centring of the velocity (egnn.py:444-445) and, in the sampler,
    // the whole reverse step incl. the centre-of-mass projection (edm.py:549-612)
    InpaintArgs ia{};
    ia.mode = io.inpaint ? 1 : 0;
    ia.eps = io.inpaint ? ws.eps : io.out; ia.nm = ws.nm; ia.z = ws.z; ia.xh0 = io.xh0;
    ia.fragment_mask = io.fragment_mask; ia.linker_mask = io.upd_linker_mask; ia.noise = io.noise; ia.rng = io.rng;
    ia.coef = e->coef_dev;
    ia.step_prep = e->step_ctr; ia.step_fin = e->step_ctr + 1; ia.T = io.T;
    ia.norm0 = io.norm0; ia.norm1 = io.norm1; ia.bias1 = io.bias1; ia.chain = io.chain;
    ia.R = io.R; ia.jump = io.jump; ia.step_tag = e->step_ctr + 2;
    if (io.R > 1) {
      if (per_mol) k_inpaint<true, true><<<B, 256, 0, st>>>(gm, ia);
      else k_inpaint<false, true><<<B, 256, 0, st>>>(gm, ia);
    } else if (per_mol) k_inpaint<true><<<B, 256, 0, st>>>(gm, ia);
    else k_inpaint<false><<<B, 256, 0, st>>>(gm, ia);
    LAUNCH_CHECK();
    e->launches += 1;
  }
  return DL_OK;
}

dl_status check_shapes(const dl_engine* e, int B, int N) {
  if (!e || !e->finalized) { set_err("engine not finalized (dl_finalize_weights)"); return DL_ERR_INVALID; }
  if (B <= 0 || N <= 0) { set_err("B and N must be positive (got %d, %d)", B, N); return DL_ERR_INVALID; }
  if ((int64_t)B * N * N > (int64_t)1 << 40) { set_err("B*N*N too large"); return DL_ERR_INVALID; }
  if (e->use_tc && e->cfg.graph_type != 0 && N > 4000) {
    set_err("cut-off graphs: N = %d exceeds the neighbour-list kernel's shared-memory staging (N <= 4000)", N);
    return DL_ERR_INVALID;
  }
  return DL_OK;
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// Device copies of a *_host entry point's arguments, in 256-byte aligned sub-buffers of the engine's stage. in() adds a
// host input (a null input gets no buffer), out() an output buffer; stage_inputs() grows the stage to fit and enqueues
// the input copies. at(i) is then buffer i's device address, or null for a null input.
struct StageLayout {
  struct Buf { const void* src; size_t bytes, off; bool used; };
  std::vector<Buf> bufs;
  size_t total = 0;
  char* base = nullptr;
  int add(const void* src, size_t bytes, bool used) {
    bufs.push_back({src, bytes, total, used});
    total += used ? align256(bytes) : 0;
    return (int)bufs.size() - 1;
  }
  int in(const void* src, size_t bytes) { return add(src, bytes, src != nullptr); }
  int out(size_t bytes) { return add(nullptr, bytes, true); }
  template <typename T> T* at(int i) const { return bufs[i].used ? reinterpret_cast<T*>(base + bufs[i].off) : nullptr; }
};

dl_status stage_inputs(HostStage& sg, StageLayout& sl, cudaStream_t st) {
  if (sg.cap < sl.total) {
    if (sg.buf) cudaFree(sg.buf);
    sg.buf = nullptr; sg.cap = 0;
    CK(cudaMalloc((void**)&sg.buf, sl.total));
    sg.cap = sl.total;
  }
  sl.base = sg.buf;
  for (const auto& b : sl.bufs)
    if (b.src) CK(cudaMemcpyAsync(sl.base + b.off, b.src, b.bytes, cudaMemcpyHostToDevice, st));
  return DL_OK;
}

// Copies a *_host call's result and its B NaN flags back, waits for them, and reports whether any flag is set.
dl_status stage_results(void* out, const void* d_out, size_t bytes, const int32_t* d_flags, int B, int32_t* nan_flags,
                        cudaStream_t st) {
  std::vector<int32_t> flags(B);
  CK(cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(flags.data(), d_flags, B * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  bool any = false;
  for (int i = 0; i < B; ++i) { any |= flags[i] != 0; if (nan_flags) nan_flags[i] = flags[i]; }
  return any ? DL_NAN_DETECTED : DL_OK;
}

// dl_set_noise_slice: the B rows of this call must lie inside the full batch
dl_status check_slice(const dl_engine* e, int B) {
  if (e->slice_B_full > 0 && e->slice_b0 + B > e->slice_B_full) {
    set_err("batch slice [%d, %d) exceeds the full batch %d", e->slice_b0, e->slice_b0 + B, e->slice_B_full);
    return DL_ERR_INVALID;
  }
  return DL_OK;
}

// Arguments every sampler entry point takes alike; has_draws: a noise tensor or the device-side stream supplies the draws.
dl_status check_sampler(const dl_engine* e, int sampler, int T, int keep_frames, bool has_draws, const float* xh,
                        const int8_t* node_mask, const float* fragment_mask, const float* linker_mask, const float* context,
                        const dl_step_coef* coef, const float* norm, const float* chain) {
  if (sampler != DL_SAMPLER_LINKER && sampler != DL_SAMPLER_INPAINT) { set_err("unknown sampler %d", sampler); return DL_ERR_INVALID; }
  if ((sampler == DL_SAMPLER_INPAINT) != (e->cfg.centering != 0)) { set_err("the inpainting sampler needs a model built with centering=1 (and vice versa)"); return DL_ERR_INVALID; }
  if (!xh || !node_mask || !fragment_mask || !linker_mask || !has_draws || !coef || !norm || !chain) {
    set_err("null argument"); return DL_ERR_INVALID;
  }
  if (T < 1 || keep_frames < 1 || keep_frames > T) { set_err("need 1 <= keep_frames <= T"); return DL_ERR_INVALID; }
  if (e->cfg.context_node_nf > 0 && !context) { set_err("context required"); return DL_ERR_INVALID; }
  return DL_OK;
}

// standard-normal draws of one chain: init + one per step + final (linker), or their masked pairs (inpainting) -- with R
// resampling passes per step, each pass's pair and, but on the last pass, the re-noise draw
uint64_t sampler_draws(int sampler, int T, int R = 1) {
  return sampler == DL_SAMPLER_INPAINT ? 1 + (uint64_t)T * (3 * R - 1) + 2 : (uint64_t)T + 2;
}

// The resampling passes of a call (dl_set_resamplings), or 0 with DL_ERR_INVALID set when the setting does not apply to it.
int call_resamplings(const dl_engine* e, int sampler, int T) {
  if (e->resamplings == 1) return 1;
  if (sampler != DL_SAMPLER_INPAINT) { set_err("resampling (dl_set_resamplings) takes DL_SAMPLER_INPAINT only"); return 0; }
  if (T != e->resample_T) {
    set_err("dl_set_resamplings was given the jump coefficients of T = %d; the call samples T = %d", e->resample_T, T);
    return 0;
  }
  return e->resamplings;
}

// Reverse steps of a call before the final one: the start step when one is set (dl_set_start_step), else T. The loop then
// runs the last loop_steps + 1 rows of the coefficient table as a chain of that length, so it also sets the draws.
// With per-molecule start steps (dl_set_start_steps) the loop runs from the largest.
int loop_steps(const dl_engine* e, int T) {
  if (e && !e->starts_t0.empty()) return *std::max_element(e->starts_t0.begin(), e->starts_t0.end());
  return e && e->start_step >= 0 ? e->start_step : T;
}

// While alive, the engine's loop runs on the sub-batch workspace and records its loop time on the ev_r* events: the
// full batch's workspace, the first loop's dl_last_elapsed_ms and the forward state dl_time_edge_kernel replays stay put.
struct SubBatchScope {
  dl_engine* e;
  const int8_t* edge_mask;
  const float* linker_mask;
  int B, N;
  int64_t mol_steps;
  explicit SubBatchScope(dl_engine* e_)
      : e(e_), edge_mask(e_->last_edge_mask), linker_mask(e_->last_linker_mask), B(e_->last_B), N(e_->last_N),
        mol_steps(e_->mol_steps) { swap(); }
  ~SubBatchScope() {
    swap();
    e->last_edge_mask = edge_mask; e->last_linker_mask = linker_mask; e->last_B = B; e->last_N = N;
    e->mol_steps = mol_steps;
  }
  void swap() { std::swap(e->ws, e->ws_sub); std::swap(e->ev_t0, e->ev_r0); std::swap(e->ev_t1, e->ev_r1); }
};

// The rows of a call with per-molecule start steps (dl_set_start_steps) in the engine's order: the caller's rows stably
// sorted by t0 descending, so that the rows a loop step computes -- those that have started -- are a prefix.
struct RowOrder {
  const float *xh, *fragment_mask, *linker_mask, *context, *alpha, *sigma;
  const int8_t *node_mask, *edge_mask, *fixed;
  RowStarts rs;
  std::vector<int> active;   // (Tl + 1) the length of the prefix loop step r computes
};

// Orders the B rows of a loop of Tl + 1 steps, stages the order, lags and scalars, and gathers the inputs (and with
// per-molecule streams the seeds, into the workspace; with fixed atoms their flags) in that order with the recovery rounds'
// gather.
dl_status order_rows(dl_engine* e, int B, int N, int Tl, const float* xh, const int8_t* node_mask, const float* fragment_mask,
                     const float* linker_mask, const int8_t* edge_mask, const float* context, const unsigned long long* seeds,
                     const int8_t* fixed, cudaStream_t st, RowOrder& ro) {
  const std::vector<int32_t>& t0 = e->starts_t0;
  std::vector<int> order(B), lag(B);
  std::vector<float> al(B), sg(B);
  for (int b = 0; b < B; ++b) order[b] = b;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return t0[a] > t0[b]; });
  for (int i = 0; i < B; ++i) {
    lag[i] = Tl - t0[order[i]]; al[i] = e->starts_alpha[order[i]]; sg[i] = e->starts_sigma[order[i]];
  }
  // row i has started at loop step r (step Tl - 1 - r) once t0 > Tl - 1 - r, i.e. lag[i] <= r; lag ascends along the order
  ro.active.resize(Tl + 1);
  for (int r = 0; r <= Tl; ++r) ro.active[r] = (int)(std::upper_bound(lag.begin(), lag.end(), r) - lag.begin());
  const bool fc_em = edge_mask && e->cfg.graph_type == DL_GRAPH_FC;
  const int xd = 3 + e->cfg.in_node_nf, C = e->cfg.context_node_nf;
  const size_t n = (size_t)B * N;
  StageLayout sl;
  const int i_src = sl.in(order.data(), B * sizeof(int)), i_lag = sl.in(lag.data(), B * sizeof(int)),
            i_al = sl.in(al.data(), B * sizeof(float)), i_sg = sl.in(sg.data(), B * sizeof(float)), i_xh = sl.out(n * xd * 4),
            i_nm = sl.out(n), i_fm = sl.out(n * 4), i_lm = sl.out(n * 4), i_em = sl.add(nullptr, n * N, fc_em),
            i_ctx = sl.add(nullptr, n * C * 4, context != nullptr && C > 0), i_fx = sl.add(nullptr, n, fixed != nullptr);
  dl_status s = stage_inputs(e->start_rows, sl, st);
  if (s != DL_OK) return s;
  RowGatherArgs ga{};
  ga.rows = sl.at<const int>(i_src); ga.N = N; ga.xd = xd; ga.C = C; ga.attempt = 0;
  ga.xh = xh; ga.fragment_mask = fragment_mask; ga.linker_mask = linker_mask; ga.context = sl.at<float>(i_ctx) ? context : nullptr;
  ga.node_mask = node_mask; ga.edge_mask = fc_em ? edge_mask : nullptr; ga.seeds = seeds;
  ga.s_xh = sl.at<float>(i_xh); ga.s_fragment_mask = sl.at<float>(i_fm); ga.s_linker_mask = sl.at<float>(i_lm);
  ga.s_context = sl.at<float>(i_ctx); ga.s_node_mask = sl.at<int8_t>(i_nm); ga.s_edge_mask = sl.at<int8_t>(i_em);
  ga.s_seeds = e->ws.seeds;
  const RowFixedArgs fa{fixed, sl.at<int8_t>(i_fx)};
  if (fixed) k_gather_rows<false><<<B, 256, 0, st>>>(ga, fa);
  else k_gather_rows<false><<<B, 256, 0, st>>>(ga);
  LAUNCH_CHECK();
  e->launches += 1;
  ro.fixed = fa.s_fixed;
  ro.xh = ga.s_xh; ro.fragment_mask = ga.s_fragment_mask; ro.linker_mask = ga.s_linker_mask; ro.context = ga.s_context;
  ro.node_mask = ga.s_node_mask; ro.edge_mask = ga.s_edge_mask;
  ro.alpha = sl.at<const float>(i_al); ro.sigma = sl.at<const float>(i_sg);
  ro.rs = RowStarts{sl.at<const int>(i_lag), sl.at<const int>(i_src), (int)n};
  return DL_OK;
}

// The fixed atoms of a sampling call (dl_set_fixed_atoms): the (B, N) flags on the device, B, N and T as set, and the
// host copy of the (T + 1, 2) scalars; flags = null: none. `vetted`: the flags are a recovery round's, gathered from a call
// whose flags were checked.
struct CallFixed {
  const int8_t* flags = nullptr;
  int B = 0, N = 0, T = 0;
  const float* scalars = nullptr;
  bool vetted = false;
  int* bad = nullptr;        // three ints of device memory for k_fixed_check and k_kept_types_check, unless vetted
};

// What dl_set_fixed_atoms set since the engine's previous sampling call, which every call reads and clears.
CallFixed take_fixed(dl_engine* e) {
  CallFixed fx;
  if (e && e->fixed_set) {
    fx.flags = reinterpret_cast<const int8_t*>(e->fixed.buf);
    fx.B = e->fixed_B; fx.N = e->fixed_N; fx.T = e->fixed_T; fx.scalars = e->fixed_scalars.data();
    fx.bad = reinterpret_cast<int*>(e->fixed.buf + align256((size_t)fx.B * fx.N));
  }
  if (e) e->fixed_set = false;
  return fx;
}

// The linker types of a sampling call (dl_set_linker_types): the B masks and the (T + 1, 2) scalars, host memory, with B
// and T as set; masks = null: none.
struct CallTypes {
  const uint32_t* masks = nullptr;
  int B = 0, T = 0;
  const float* scalars = nullptr;
};

// What dl_set_linker_types set since the engine's previous sampling call, which every call reads and clears.
CallTypes take_types(dl_engine* e) {
  CallTypes ty;
  if (e && e->types_set) {
    ty.masks = e->types_masks.data(); ty.B = e->types_B; ty.T = e->types_T; ty.scalars = e->types_scalars.data();
  }
  if (e) e->types_set = false;
  return ty;
}

// Captures one reverse step over the first Bp rows of the workspace into *graph.
dl_status capture_step(dl_engine* e, int Bp, int N, const FwdIO& io, cudaStream_t st, cudaGraph_t* graph) {
  CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const dl_status s = enqueue_forward(e, Bp, N, io, st);
  const cudaError_t ce = cudaStreamEndCapture(st, graph);
  if (s != DL_OK) { if (*graph) cudaGraphDestroy(*graph); *graph = nullptr; return s; }
  if (ce != cudaSuccess) { set_err("cudaStreamEndCapture -> %s", cudaGetErrorString(ce)); return DL_ERR_CUDA; }
  return DL_OK;
}

}  // namespace

extern "C" {

const char* dl_version(void) { return "difflinker_b200 0.1 (sm_90a)"; }
const char* dl_last_error(void) { return g_err; }

dl_status dl_create(const dl_config* cfg, dl_engine** out) { return dl_create_ex(cfg, nullptr, out); }

dl_status dl_create_ex(const dl_config* cfg, const dl_egnn_options* opts, dl_engine** out) {
  if (!cfg || !out) { set_err("null argument"); return DL_ERR_INVALID; }
  const dl_egnn_options o = opts ? *opts : dl_egnn_options{0, 15.0f, 0, DL_AGGR_SUM};
  if (o.sin_embedding != 0 && o.sin_embedding != 1) { set_err("sin_embedding must be 0 or 1 (got %d)", o.sin_embedding); return DL_ERR_INVALID; }
  if (o.tanh != 0 && o.tanh != 1) { set_err("tanh must be 0 or 1 (got %d)", o.tanh); return DL_ERR_INVALID; }
  if (o.aggregation != DL_AGGR_SUM && o.aggregation != DL_AGGR_MEAN) { set_err("unknown aggregation %d", o.aggregation); return DL_ERR_INVALID; }
  if (!std::isfinite(o.coords_range)) { set_err("coords_range must be finite"); return DL_ERR_INVALID; }
  if (cfg->hidden_nf != H) { set_err("hidden_nf must be %d (got %d)", H, cfg->hidden_nf); return DL_ERR_UNSUPPORTED; }
  if (cfg->n_dims != 3) { set_err("n_dims must be 3"); return DL_ERR_UNSUPPORTED; }
  const int D = cfg->in_node_nf + cfg->context_node_nf + (cfg->condition_time ? 1 : 0);
  if (D > MAX_DIN || cfg->in_node_nf < 1 || 3 + cfg->in_node_nf > MAX_XHD) {
    set_err("unsupported feature widths F=%d C=%d", cfg->in_node_nf, cfg->context_node_nf);
    return DL_ERR_UNSUPPORTED;
  }
  if (cfg->n_layers < 1 || cfg->inv_sublayers < 1) { set_err("n_layers/inv_sublayers must be >= 1"); return DL_ERR_INVALID; }
  if (cfg->graph_type < 0 || cfg->graph_type > 3) { set_err("bad graph_type"); return DL_ERR_INVALID; }
  if (cfg->graph_type != DL_GRAPH_FC && cfg->context_node_nf < 2) {
    set_err("pocket graphs need fragment_only/pocket_only context columns"); return DL_ERR_INVALID;
  }
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  if (cfg->device < 0 || cfg->device >= ndev) { set_err("device %d not available (%d devices)", cfg->device, ndev); return DL_ERR_INVALID; }
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) {
    set_err("difflinker_b200 is built for sm_90a only; device is sm_%d%d", prop.major, prop.minor);
    return DL_ERR_UNSUPPORTED;
  }
  dl_engine* e = new dl_engine();
  e->cfg = *cfg;
  e->opts = o;
  e->D = D;
  e->num_sms = prop.multiProcessorCount;
  e->max_threads_per_sm = prop.maxThreadsPerMultiProcessor;
  e->use_tc = tc::AVAILABLE && cfg->edge_impl != DL_EDGE_SIMT;
  CK(cudaStreamCreateWithFlags(&e->loop_stream, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&e->ev_out, cudaEventDisableTiming));
  CK(cudaEventCreate(&e->ev_t0));
  CK(cudaEventCreate(&e->ev_t1));
  CK(cudaEventCreate(&e->ev_r0));
  CK(cudaEventCreate(&e->ev_r1));
  CK(cudaEventCreate(&e->ev_g0));
  CK(cudaEventCreate(&e->ev_g1));
  CK(cudaMalloc((void**)&e->step_ctr, 3 * sizeof(int)));
  CK(cudaFuncSetAttribute(k_node<ACT_SILU>, cudaFuncAttributeMaxDynamicSharedMemorySize, 3 * NODE_TM * LDX * sizeof(float)));
  CK(opt_in_edge_simt<true>());
  CK(opt_in_edge_simt<false>());
  CK(cudaFuncSetAttribute(k_nbr, cudaFuncAttributeMaxDynamicSharedMemorySize, 4000 * CUT_SMEM_PER_NODE));
  if (getenv("DL_TIME_KERNELS")) e->times.on = true;
  if (const char* v = getenv("DL_WAIT_MODE")) { const int m = atoi(v); cudaMemcpyToSymbol(tc::c_wait_mode, &m, sizeof(int)); }
  if (const char* v = getenv("DL_CHAIN_OVERLAP")) chain_overlap_enabled() = atoi(v) != 0;   // 0: plain stream order between kernels
  dl_status s = tc::configure();
  if (s == DL_OK) s = tcn::configure_node();
  if (s != DL_OK) { set_err("cudaFuncSetAttribute failed for the tensor-core kernels"); delete e; return s; }
  *out = e;
  return DL_OK;
}

dl_status dl_destroy(dl_engine* e) {
  if (!e) return DL_OK;
  e->times.report();
  cudaSetDevice(e->cfg.device);
  cudaDeviceSynchronize();
  free_workspace(e->ws);
  free_workspace(e->ws_sub);
  if (e->sub_rows.buf) cudaFree(e->sub_rows.buf);
  if (e->start_rows.buf) cudaFree(e->start_rows.buf);
  if (e->hashes.buf) cudaFree(e->hashes.buf);
  if (e->ring_masks.buf) cudaFree(e->ring_masks.buf);
  if (e->anchors.buf) cudaFree(e->anchors.buf);
  if (e->fixed.buf) cudaFree(e->fixed.buf);
  if (e->wblob) cudaFree(e->wblob);
  if (e->wblob_tc) cudaFree(e->wblob_tc);
  if (e->coef_dev) cudaFree(e->coef_dev);
  if (e->step_ctr) cudaFree(e->step_ctr);
  if (e->guide_clash) cudaFree(e->guide_clash);
  if (e->stage.buf) cudaFree(e->stage.buf);
  if (e->loop_stream) cudaStreamDestroy(e->loop_stream);
  if (e->ev_in) cudaEventDestroy(e->ev_in);
  if (e->ev_out) cudaEventDestroy(e->ev_out);
  if (e->ev_t0) cudaEventDestroy(e->ev_t0);
  if (e->ev_t1) cudaEventDestroy(e->ev_t1);
  for (cudaEvent_t ev : {e->ev_r0, e->ev_r1, e->ev_g0, e->ev_g1}) if (ev) cudaEventDestroy(ev);
  delete e;
  return DL_OK;
}

int64_t dl_expected_param_count(const dl_engine* e) {
  if (!e) return 0;
  int64_t n = 0;
  for (auto& p : expected_params(e->cfg, edges_in(e))) n += p.numel;
  return n;
}

dl_status dl_set_weight(dl_engine* e, const char* name, const float* data, int64_t numel) {
  if (!e || !name || !data) { set_err("null argument"); return DL_ERR_INVALID; }
  for (auto& p : expected_params(e->cfg, edges_in(e))) {
    if (p.name == name) {
      if (p.numel != numel) {
        set_err("weight %s: expected %lld elements, got %lld", name, (long long)p.numel, (long long)numel);
        return DL_ERR_WEIGHTS;
      }
      e->raw[p.name].assign(data, data + numel);
      e->finalized = false;
      return DL_OK;
    }
  }
  set_err("unexpected weight name %s", name);
  return DL_ERR_WEIGHTS;
}

dl_status dl_finalize_weights(dl_engine* e) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  for (auto& p : expected_params(e->cfg, edges_in(e)))
    if (!e->raw.count(p.name)) { set_err("missing weight %s", p.name.c_str()); return DL_ERR_WEIGHTS; }
  const int L = e->cfg.n_layers, S = e->cfg.inv_sublayers, D = e->D;
  const RawWeights& raw = e->raw;
  Packer pk;
  e->gcl.assign(L * S, GclW{});
  e->eq.assign(L, EqW{});
  pk.add(&e->We_t, transpose_block(raw.at("dynamics.embedding.weight"), H, D, 0, D));
  pk.add(&e->be, raw.at("dynamics.embedding.bias"));
  pk.add(&e->Wo, raw.at("dynamics.embedding_out.weight"));
  pk.add(&e->bo, raw.at("dynamics.embedding_out.bias"));
  char buf[160];
  for (int l = 0; l < L; ++l) {
    for (int s = 0; s < S; ++s) {
      snprintf(buf, sizeof(buf), "dynamics.e_block_%d.gcl_%d.", l, s);
      const std::string p(buf);
      GclW& w = e->gcl[l * S + s];
      pack_gcl(pk, w, raw, p, 2 * H + edges_in(e));
      pack_edge_mlp_denoiser(pk, w, raw, p + "edge_mlp.", e->opts.sin_embedding != 0);
      pk.add_tc(&w.W3_tc, tcn::pack_blocks(raw.at(p + "node_mlp.0.weight"), 2 * H, 2, pk.tc, &w.w3_descale));
      pk.add_tc(&w.W4_tc, tcn::pack_blocks(raw.at(p + "node_mlp.2.weight"), H, 1, pk.tc, &w.w4_descale));
    }
    snprintf(buf, sizeof(buf), "dynamics.e_block_%d.gcl_equiv.coord_mlp.", l);
    const std::string p(buf);
    EqW& q = e->eq[l];
    pack_edge_mlp(pk, q, raw, p, 2 * H + edges_in(e));
    pack_edge_mlp_denoiser(pk, q, raw, p, e->opts.sin_embedding != 0);
    pk.add(&q.w5, raw.at(p + "4.weight"));
  }
  dl_status s = upload_blob(pk.blob, &e->wblob);
  if (s == DL_OK) s = upload_blob(pk.tc, &e->wblob_tc);
  if (s != DL_OK) return s;
  pk.point(e->wblob, e->wblob_tc);
  e->finalized = true;
  return DL_OK;
}

dl_status dl_dynamics_forward(dl_engine* e, int32_t B, int32_t N, const float* t, int32_t t_numel, const float* xh,
                              const int8_t* node_mask, const float* linker_mask, const int8_t* edge_mask,
                              const float* context, float* out, int32_t* nan_flags, void* stream) {
  dl_status s = check_shapes(e, B, N);
  if (s != DL_OK) return s;
  if (!xh || !node_mask || !out) { set_err("xh/node_mask/out must not be null"); return DL_ERR_INVALID; }
  if (e->cfg.condition_time && (!t || (t_numel != 1 && t_numel != B))) { set_err("t must hold 1 or B values"); return DL_ERR_INVALID; }
  if (e->cfg.context_node_nf > 0 && !context) { set_err("context required (context_node_nf=%d)", e->cfg.context_node_nf); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if ((s = ensure_workspace(e, B, N)) != DL_OK) return s;
  CK(cudaEventRecord(e->ev_t0, st));
  if (nan_flags) CK(cudaMemsetAsync(nan_flags, 0, B * sizeof(int32_t), st));
  if ((s = build_forward_plan(e, B, N, node_mask, linker_mask, edge_mask, st)) != DL_OK) return s;
  FwdIO io;
  io.xh = xh; io.t = t; io.t_numel = t_numel; io.out = out; io.node_mask = node_mask; io.linker_mask = linker_mask;
  io.edge_mask = edge_mask; io.context = context; io.nan_flags = nan_flags;
  if ((s = enqueue_forward(e, B, N, io, st)) != DL_OK) return s;
  CK(cudaEventRecord(e->ev_t1, st));
  e->times.collect(st);
  return DL_OK;
}

dl_status dl_dynamics_forward_host(dl_engine* e, int32_t B, int32_t N, const float* t, int32_t t_numel,
                                   const float* xh, const int8_t* node_mask, const float* linker_mask,
                                   const int8_t* edge_mask, const float* context, float* out, int32_t* nan_flags) {
  dl_status s = check_shapes(e, B, N);
  if (s != DL_OK) return s;
  CK(cudaSetDevice(e->cfg.device));
  const size_t n = (size_t)B * N, xh_bytes = n * (3 + e->cfg.in_node_nf) * 4;
  const bool fc_em = edge_mask && e->cfg.graph_type == DL_GRAPH_FC;
  StageLayout sl;
  const int i_t = sl.in(t, sizeof(float) * t_numel), i_xh = sl.in(xh, xh_bytes), i_nm = sl.in(node_mask, n),
            i_lm = sl.in(linker_mask, n * 4), i_em = sl.in(fc_em ? edge_mask : nullptr, n * N),
            i_ctx = sl.in(context, n * e->cfg.context_node_nf * 4), i_out = sl.out(xh_bytes), i_fl = sl.out(B * 4);
  cudaStream_t st = e->loop_stream;
  if ((s = stage_inputs(e->stage, sl, st)) != DL_OK) return s;
  s = dl_dynamics_forward(e, B, N, sl.at<const float>(i_t), t_numel, sl.at<const float>(i_xh), sl.at<const int8_t>(i_nm),
                          sl.at<const float>(i_lm), sl.at<const int8_t>(i_em), sl.at<const float>(i_ctx),
                          sl.at<float>(i_out), sl.at<int32_t>(i_fl), st);
  if (s != DL_OK) return s;
  return stage_results(out, sl.at<float>(i_out), xh_bytes, sl.at<int32_t>(i_fl), B, nan_flags, st);
}

// torch's launch geometry for randn(numel) on this device (see NoiseRng)
static void randn_geometry(const dl_engine* e, long long numel, int* S, unsigned long long* consumed) {
  long long grid = (numel + 255) / 256;
  grid = std::min<long long>(grid, (long long)e->num_sms * (e->max_threads_per_sm / 256));
  grid = std::max<long long>(grid, 1);
  *S = (int)(256 * grid);
  *consumed = (unsigned long long)(((numel - 1) / (4LL * *S) + 1) * 4);
}
static NoiseRng make_rng(const dl_engine* e, int B, int N, uint64_t seed, uint64_t offset) {
  NoiseRng q{};
  const int F = e->cfg.in_node_nf;
  unsigned long long cx = 0, ch = 0;
  const int B_full = e->slice_B_full > 0 ? e->slice_B_full : B;   // geometry of the FULL batch's randn calls
  randn_geometry(e, (long long)B_full * N * 3, &q.Sx, &cx);
  randn_geometry(e, (long long)B_full * N * F, &q.Sh, &ch);
  q.seed = seed; q.offset = offset; q.cx = cx; q.per_draw = cx + ch; q.F = F; q.on = NOISE_BATCH;
  q.g0 = e->slice_B_full > 0 ? e->slice_b0 * N : 0;
  return q;
}

static dl_status sample_chain_impl(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                   const float* xh, const int8_t* node_mask, const float* fragment_mask,
                                   const float* linker_mask, const int8_t* edge_mask, const float* context,
                                   const float* noise, const NoiseRng* rng, const dl_step_coef* coef, const float* norm,
                                   float* chain, int32_t* nan_flags, void* stream, const CallFixed& fx,
                                   const CallTypes& ty);

dl_status dl_sample_chain(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                          const float* xh, const int8_t* node_mask, const float* fragment_mask,
                          const float* linker_mask, const int8_t* edge_mask, const float* context,
                          const float* noise, const dl_step_coef* coef, const float* norm, float* chain,
                          int32_t* nan_flags, void* stream) {
  const CallFixed fx = take_fixed(e);
  const CallTypes ty = take_types(e);
  if (!noise) { set_err("null argument (noise): use dl_sample_chain_rng to draw on the device"); return DL_ERR_INVALID; }
  return sample_chain_impl(e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask, linker_mask, edge_mask, context, noise,
                           nullptr, coef, norm, chain, nan_flags, stream, fx, ty);
}

dl_status dl_sample_chain_rng(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                              const float* xh, const int8_t* node_mask, const float* fragment_mask,
                              const float* linker_mask, const int8_t* edge_mask, const float* context, uint64_t seed,
                              uint64_t offset, uint64_t* offset_consumed, const dl_step_coef* coef, const float* norm,
                              float* chain, int32_t* nan_flags, void* stream) {
  const CallFixed fx = take_fixed(e);
  const CallTypes ty = take_types(e);
  dl_status s = check_shapes(e, B, N);
  if (s == DL_OK) s = check_slice(e, B);
  if (s != DL_OK) return s;
  if (offset % 4 != 0) { set_err("philox offset must be a multiple of 4 (torch.Generator.get_offset())"); return DL_ERR_INVALID; }
  if (!e->starts_t0.empty()) {
    set_err("dl_sample_chain_rng: the batch stream's draws are not per molecule, so it takes no per-molecule start steps "
            "(dl_set_start_steps): use dl_sample_chain_seeded or a noise tensor");
    return DL_ERR_INVALID;
  }
  const int R = call_resamplings(e, sampler, T);
  if (R < 1) return DL_ERR_INVALID;
  const NoiseRng q = make_rng(e, B, N, seed, offset);
  if (offset_consumed) *offset_consumed = sampler_draws(sampler, loop_steps(e, T), R) * q.per_draw;
  return sample_chain_impl(e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask, linker_mask, edge_mask, context, nullptr,
                           &q, coef, norm, chain, nan_flags, stream, fx, ty);
}

}  // extern "C"

// dl_sample_chain_seeded with the fixed atoms fx and the linker types ty: the recovery rounds' entry, which passes their
// gathered flags and masks.
static dl_status sample_seeded(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                               const float* xh, const int8_t* node_mask, const float* fragment_mask, const float* linker_mask,
                               const int8_t* edge_mask, const float* context, const uint64_t* seeds, const dl_step_coef* coef,
                               const float* norm, float* chain, int32_t* nan_flags, void* stream, const CallFixed& fx,
                               const CallTypes& ty) {
  // the seeds name the molecules, so the engine's batch slice does not apply; sample_chain_impl copies them into the
  // workspace and points the stream at that copy
  NoiseRng q{};
  q.seeds = reinterpret_cast<const unsigned long long*>(seeds);
  q.F = e ? e->cfg.in_node_nf : 0; q.N = N; q.on = NOISE_PER_MOLECULE;
  return sample_chain_impl(e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask, linker_mask, edge_mask, context, nullptr,
                           &q, coef, norm, chain, nan_flags, stream, fx, ty);
}

extern "C" {

dl_status dl_sample_chain_seeded(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                 const float* xh, const int8_t* node_mask, const float* fragment_mask,
                                 const float* linker_mask, const int8_t* edge_mask, const float* context,
                                 const uint64_t* seeds, const dl_step_coef* coef, const float* norm, float* chain,
                                 int32_t* nan_flags, void* stream) {
  return sample_seeded(e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask, linker_mask, edge_mask, context, seeds,
                       coef, norm, chain, nan_flags, stream, take_fixed(e), take_types(e));
}

dl_status dl_set_noise_slice(dl_engine* e, int32_t B_full, int32_t b0) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  if (B_full < 0 || b0 < 0 || (B_full > 0 && b0 >= B_full)) { set_err("bad batch slice (%d of %d)", b0, B_full); return DL_ERR_INVALID; }
  e->slice_B_full = B_full; e->slice_b0 = B_full > 0 ? b0 : 0;
  return DL_OK;
}

dl_status dl_set_start_step(dl_engine* e, int32_t t0, float alpha_t0, float sigma_t0) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  if (t0 < 0) { e->start_step = -1; e->start_alpha = e->start_sigma = 0.f; return DL_OK; }
  if (!std::isfinite(alpha_t0) || !std::isfinite(sigma_t0)) { set_err("alpha_t0 and sigma_t0 must be finite"); return DL_ERR_INVALID; }
  e->start_step = t0; e->start_alpha = alpha_t0; e->start_sigma = sigma_t0;
  e->starts_t0.clear(); e->starts_alpha.clear(); e->starts_sigma.clear();
  return DL_OK;
}

dl_status dl_set_start_steps(dl_engine* e, int32_t B, const int32_t* t0, const float* alpha, const float* sigma) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  if (B < 0) { set_err("dl_set_start_steps: B must be >= 0 (got %d)", B); return DL_ERR_INVALID; }
  if (B > 0 && (!t0 || !alpha || !sigma)) { set_err("dl_set_start_steps: null t0, alpha or sigma"); return DL_ERR_INVALID; }
  for (int b = 0; b < B; ++b) {
    if (t0[b] < 0) { set_err("dl_set_start_steps: t0[%d] = %d is negative", b, t0[b]); return DL_ERR_INVALID; }
    if (!std::isfinite(alpha[b]) || !std::isfinite(sigma[b])) {
      set_err("dl_set_start_steps: alpha[%d] and sigma[%d] must be finite", b, b);
      return DL_ERR_INVALID;
    }
  }
  e->starts_t0.assign(t0, t0 + B); e->starts_alpha.assign(alpha, alpha + B); e->starts_sigma.assign(sigma, sigma + B);
  e->start_step = -1; e->start_alpha = e->start_sigma = 0.f;
  return DL_OK;
}

dl_status dl_set_resamplings(dl_engine* e, int32_t r, int32_t T, const float* jump) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  if (r < 1) { set_err("dl_set_resamplings: r must be >= 1 (got %d)", r); return DL_ERR_INVALID; }
  if (r == 1) { e->resamplings = 1; e->resample_T = 0; e->jump.clear(); return DL_OK; }
  if (!jump) { set_err("dl_set_resamplings: r = %d needs the jump coefficients", r); return DL_ERR_INVALID; }
  if (T < 1) { set_err("dl_set_resamplings: T must be >= 1 (got %d)", T); return DL_ERR_INVALID; }
  if ((int64_t)T * r > (1 << 24)) {   // the expanded coefficient table and the draw indices stay well inside int
    set_err("dl_set_resamplings: T * r = %lld passes exceeds 2^24", (long long)T * r);
    return DL_ERR_INVALID;
  }
  for (int i = 0; i < 2 * T; ++i)
    if (!std::isfinite(jump[i])) {
      set_err("dl_set_resamplings: jump[%d][%d] is not finite", i / 2, i % 2);
      return DL_ERR_INVALID;
    }
  e->resamplings = r; e->resample_T = T; e->jump.assign(jump, jump + 2 * T);
  return DL_OK;
}

dl_status dl_set_clash_guidance(dl_engine* e, float scale, int32_t steps, int32_t n_types, const float* clash) {
  if (!e) { set_err("dl_set_clash_guidance: null engine"); return DL_ERR_INVALID; }
  const char* why = nullptr;
  if (!std::isfinite(scale) || scale < 0.f) why = "scale must be finite and >= 0";
  else if (steps < 0) why = "steps must be >= 0";
  if (why) { set_err("dl_set_clash_guidance: %s (got scale %g, steps %d)", why, (double)scale, steps); return DL_ERR_INVALID; }
  if (steps == 0 || scale == 0.f) { e->guide_scale = 0.f; e->guide_steps = e->guide_types = 0; return DL_OK; }
  if (n_types < 1 || !clash) { set_err("dl_set_clash_guidance: needs n_types >= 1 and a clash table"); return DL_ERR_INVALID; }
  // a host copy: the calls already enqueued keep the table they uploaded, later calls upload this one
  e->guide_table.assign(clash, clash + (size_t)n_types * n_types);
  e->guide_scale = scale; e->guide_steps = steps; e->guide_types = n_types;
  return DL_OK;
}

dl_status dl_set_solver(dl_engine* e, int32_t kind, int32_t T, const float* table) {
  if (!e) { set_err("dl_set_solver: null engine"); return DL_ERR_INVALID; }
  if (kind != DL_SOLVER_ANCESTRAL && kind != DL_SOLVER_DDIM && kind != DL_SOLVER_DPMPP_2M) {
    set_err("dl_set_solver: unknown kind %d", kind);
    return DL_ERR_INVALID;
  }
  if (kind == DL_SOLVER_ANCESTRAL) { e->solver_kind = kind; e->solver_T = 0; e->solver_table.clear(); return DL_OK; }
  if (!table) { set_err("dl_set_solver: kind %d needs its table", kind); return DL_ERR_INVALID; }
  if (T < 1 || T > (1 << 24)) { set_err("dl_set_solver: T must lie in [1, 2^24] (got %d)", T); return DL_ERR_INVALID; }
  for (int i = 0; i < 8 * (T + 1); ++i)
    if (!std::isfinite(table[i])) {
      set_err("dl_set_solver: table[%d][%d] is not finite", i / 8, i % 8);
      return DL_ERR_INVALID;
    }
  for (int r = 0; r < T; ++r)
    if (!(table[8 * r + 6] > 0.f)) {
      set_err("dl_set_solver: row %d has h = %g <= 0 (a grid point repeats)", r, (double)table[8 * r + 6]);
      return DL_ERR_INVALID;
    }
  // a host copy: the calls already enqueued keep the rows they uploaded, later calls upload this table
  e->solver_kind = kind; e->solver_T = T; e->solver_table.assign(table, table + 8 * (size_t)(T + 1));
  return DL_OK;
}

dl_status dl_set_ring_sizes(dl_engine* e, uint64_t allowed) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  if (allowed & 7u) {
    set_err("dl_set_ring_sizes: bits 0-2 of allowed must be clear (a ring has at least 3 atoms; got 0x%llx)",
            (unsigned long long)allowed);
    return DL_ERR_INVALID;
  }
  e->ring_allowed = allowed;
  e->ring_set = true;
  return DL_OK;
}

dl_status dl_set_anchors(dl_engine* e, int32_t B, int32_t N, const int8_t* anchors, void* stream) {
  const char* why = nullptr;
  if (!e) why = "null engine";
  else if (B < 1 || N < 1) why = "B and N must be >= 1";
  else if (!anchors) why = "null anchors";
  if (why) { set_err("dl_set_anchors: %s", why); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  e->anchors_set = false;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  StageLayout al;
  const int i_an = al.out((size_t)B * N);
  dl_status s = stage_inputs(e->anchors, al, st);
  if (s != DL_OK) return s;
  CK(cudaMemcpyAsync(al.at<int8_t>(i_an), anchors, (size_t)B * N, cudaMemcpyDefault, st));
  e->anchors_set = true;
  e->anchors_B = B;
  e->anchors_N = N;
  return DL_OK;
}

dl_status dl_set_fixed_atoms(dl_engine* e, int32_t B, int32_t N, const int8_t* fixed, int32_t T, const float* scalars,
                             void* stream) {
  if (!e) { set_err("dl_set_fixed_atoms: null engine"); return DL_ERR_INVALID; }
  e->fixed_set = false;
  if (!fixed) return DL_OK;
  const char* why = nullptr;
  if (B < 1 || N < 1) why = "B and N must be >= 1";
  else if (T < 1 || T > (1 << 24)) why = "T must lie in [1, 2^24]";
  else if (!scalars) why = "null scalars";
  if (why) { set_err("dl_set_fixed_atoms: %s", why); return DL_ERR_INVALID; }
  for (int i = 0; i < 2 * (T + 1); ++i)
    if (!std::isfinite(scalars[i])) {
      set_err("dl_set_fixed_atoms: scalars[%d][%d] is not finite", i / 2, i % 2);
      return DL_ERR_INVALID;
    }
  CK(cudaSetDevice(e->cfg.device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  StageLayout fl;
  const int i_fx = fl.out((size_t)B * N);
  fl.out(3 * sizeof(int));   // the call's vetting (k_fixed_check, k_kept_types_check)
  dl_status s = stage_inputs(e->fixed, fl, st);
  if (s != DL_OK) return s;
  CK(cudaMemcpyAsync(fl.at<int8_t>(i_fx), fixed, (size_t)B * N, cudaMemcpyDefault, st));
  e->fixed_scalars.assign(scalars, scalars + 2 * (size_t)(T + 1));
  e->fixed_set = true;
  e->fixed_B = B; e->fixed_N = N; e->fixed_T = T;
  return DL_OK;
}

dl_status dl_set_linker_types(dl_engine* e, int32_t B, int32_t F, const uint32_t* masks, int32_t T, const float* scalars) {
  if (!e) { set_err("dl_set_linker_types: null engine"); return DL_ERR_INVALID; }
  e->types_set = false;
  if (!masks) return DL_OK;
  const char* why = nullptr;
  if (B < 1) why = "B must be >= 1";
  else if (F != e->cfg.in_node_nf) why = "F must be the model's number of type channels (dl_config.in_node_nf)";
  else if (T < 1 || T > (1 << 24)) why = "T must lie in [1, 2^24]";
  else if (!scalars) why = "null scalars";
  if (why) { set_err("dl_set_linker_types: %s", why); return DL_ERR_INVALID; }
  for (int b = 0; b < B; ++b) {
    if (masks[b] == 0 || (F < 32 && (masks[b] >> F) != 0)) {
      set_err("dl_set_linker_types: the mask of molecule %d, 0x%x, %s", b, masks[b],
              masks[b] == 0 ? "allows no type" : "has bits at or above F");
      return DL_ERR_INVALID;
    }
  }
  for (int i = 0; i < 2 * (T + 1); ++i)
    if (!std::isfinite(scalars[i])) {
      set_err("dl_set_linker_types: scalars[%d][%d] is not finite", i / 2, i % 2);
      return DL_ERR_INVALID;
    }
  e->types_masks.assign(masks, masks + B);
  e->types_scalars.assign(scalars, scalars + 2 * (size_t)(T + 1));
  e->types_set = true;
  e->types_B = B; e->types_T = T;
  return DL_OK;
}

dl_status dl_noise_fill(dl_engine* e, int32_t n_draws, int32_t B, int32_t N, uint64_t seed, uint64_t offset, float* out,
                        uint64_t* offset_consumed, void* stream) {
  dl_status s = check_shapes(e, B, N);
  if (s != DL_OK) return s;
  if (!out || n_draws < 1) { set_err("null argument"); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  const NoiseRng q = make_rng(e, B, N, seed, offset);
  if (offset_consumed) *offset_consumed = (uint64_t)n_draws * q.per_draw;
  k_noise_fill<<<e->num_sms * 4, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(n_draws, B * N, 3 + e->cfg.in_node_nf, q, out);
  LAUNCH_CHECK();
  return DL_OK;
}

dl_status dl_noise_fill_inpaint(dl_engine* e, int32_t T, int32_t B, int32_t N, const int8_t* node_mask,
                                const float* fragment_mask, uint64_t seed, uint64_t offset, float* out,
                                uint64_t* offset_consumed, void* stream) {
  dl_status s = check_shapes(e, B, N);
  if (s != DL_OK) return s;
  if (!node_mask || !fragment_mask || !out) { set_err("null argument"); return DL_ERR_INVALID; }
  if (T < 1 || 2 * T + 3 > 65535) { set_err("need 1 <= T <= 32766 (got %d)", T); return DL_ERR_INVALID; }
  if ((s = check_slice(e, B)) != DL_OK) return s;
  const int R = call_resamplings(e, DL_SAMPLER_INPAINT, T);
  if (R < 1) return DL_ERR_INVALID;
  const uint64_t draws = sampler_draws(DL_SAMPLER_INPAINT, T, R);
  if (draws > 65535) { set_err("%llu draws exceed the grid's 65535 rows", (unsigned long long)draws); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  const NoiseRng q = make_rng(e, B, N, seed, offset);
  if (offset_consumed) *offset_consumed = draws * q.per_draw;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (R > 1)
    k_com_free_draws<false, true><<<dim3(B, (unsigned)draws), 256, 0, st>>>(N, 3 + e->cfg.in_node_nf, T, q, node_mask,
                                                                           fragment_mask, out, R);
  else
    k_com_free_draws<false><<<dim3(B, 2 * T + 3), 256, 0, st>>>(N, 3 + e->cfg.in_node_nf, T, q, node_mask, fragment_mask, out);
  LAUNCH_CHECK();
  return DL_OK;
}

static dl_status sample_chain_impl(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                   const float* xh, const int8_t* node_mask, const float* fragment_mask,
                                   const float* linker_mask, const int8_t* edge_mask, const float* context,
                                   const float* noise, const NoiseRng* rng, const dl_step_coef* coef, const float* norm,
                                   float* chain, int32_t* nan_flags, void* stream, const CallFixed& fx,
                                   const CallTypes& ty) {
  const bool per_mol = rng && rng->on == NOISE_PER_MOLECULE;
  dl_status s = check_shapes(e, B, N);
  if (s == DL_OK) s = check_sampler(e, sampler, T, keep_frames, noise || (rng && (!per_mol || rng->seeds)), xh, node_mask,
                                    fragment_mask, linker_mask, context, coef, norm, chain);
  if (s != DL_OK) return s;
  const bool inpaint = sampler == DL_SAMPLER_INPAINT;
  const bool partial = e->start_step >= 0;
  const bool per_row = !e->starts_t0.empty();   // per-molecule start steps (dl_set_start_steps)
  if (partial && inpaint) { set_err("the inpainting sampler takes no start step (dl_set_start_step)"); return DL_ERR_INVALID; }
  if (partial && e->start_step > T) { set_err("start step %d exceeds T = %d", e->start_step, T); return DL_ERR_INVALID; }
  if (per_row) {
    if ((int)e->starts_t0.size() != B) {
      set_err("per-molecule start steps were set for %d molecules; the call samples %d", (int)e->starts_t0.size(), B);
      return DL_ERR_INVALID;
    }
    if (inpaint) { set_err("the inpainting sampler takes no start steps (dl_set_start_steps)"); return DL_ERR_INVALID; }
    if (rng && !per_mol) { set_err("the batch stream takes no per-molecule start steps"); return DL_ERR_INVALID; }
    if (loop_steps(e, T) > T) { set_err("start step %d exceeds T = %d", loop_steps(e, T), T); return DL_ERR_INVALID; }
  }
  const int R = call_resamplings(e, sampler, T);
  if (R < 1) return DL_ERR_INVALID;
  if (e->guide_steps > 0) {
    const char* why = nullptr;
    if (inpaint) why = "the inpainting sampler re-noises the pocket";
    else if (partial || per_row) why = "it takes no start step (dl_set_start_step, dl_set_start_steps)";
    else if (e->cfg.graph_type == DL_GRAPH_FC) why = "DL_GRAPH_FC has no pocket rows";
    else if (e->guide_steps > T) why = "its steps exceed the call's T";
    else if (e->guide_types > e->cfg.in_node_nf) why = "its table has more atom types than the model's features";
    else if (N > CONN_MAX_N) why = "it takes N <= 8192";
    else if (!context || e->cfg.context_node_nf < 1) why = "it needs the context's pocket column";
    if (why) {
      set_err("clash guidance (dl_set_clash_guidance): %s", why);
      return DL_ERR_INVALID;
    }
  }
  const bool ode = e->solver_kind != DL_SOLVER_ANCESTRAL;
  if (ode && (inpaint || T != e->solver_T)) {
    if (inpaint) set_err("dl_set_solver takes DL_SAMPLER_LINKER only");
    else set_err("dl_set_solver was given the table of T = %d; the call samples T = %d", e->solver_T, T);
    return DL_ERR_INVALID;
  }
  const bool fix = fx.flags != nullptr;
  if (fix && (inpaint || B != fx.B || N != fx.N || T != fx.T)) {
    if (inpaint) set_err("dl_set_fixed_atoms takes DL_SAMPLER_LINKER only: the inpainting sampler re-noises every atom");
    else set_err("dl_set_fixed_atoms was given B = %d, N = %d, T = %d; the call samples B = %d, N = %d, T = %d", fx.B, fx.N,
                 fx.T, B, N, T);
    return DL_ERR_INVALID;
  }
  const bool types = ty.masks != nullptr;
  if (types && (inpaint || B != ty.B || T != ty.T)) {
    if (inpaint) set_err("dl_set_linker_types takes DL_SAMPLER_LINKER only: the inpainting sampler updates every atom");
    else set_err("dl_set_linker_types was given B = %d, T = %d; the call samples B = %d, T = %d", ty.B, ty.T, B, T);
    return DL_ERR_INVALID;
  }
  // A start step t0 runs the table's last t0 + 1 rows -- steps t0-1 .. 0, then the final one -- as a loop of Tl = t0 steps:
  // loop step r reads row r of the copied rows and draw r + 1, so the draws are eps, one per step and the final one.
  const int Tl = loop_steps(e, T);
  coef += T - Tl;
  static_assert(sizeof(dl_step_coef) == 32, "dl_step_coef layout");
  // Resampling: the loop runs P = T*R passes and the final step. Pass k*R + u reads row k of the caller's table, whose frame
  // only its last pass writes; the jump coefficients follow the table on the device. A solver (never with R > 1, which is
  // the inpainting sampler's) puts the same rows of its table there instead.
  const int P = Tl * R, rows = P + 1;
  // Fixed atoms put the (alpha_s, sigma_s) of the loop's Tl steps after them, linker types the (alpha_t, sigma_t) of its
  // rows and then the B masks.
  const size_t coef_bytes = (size_t)rows * sizeof(dl_step_coef) + (R > 1 ? e->jump.size() * sizeof(float) : 0) +
                            (ode ? (size_t)rows * 8 * sizeof(float) : 0) + (fix ? (size_t)Tl * 2 * sizeof(float) : 0) +
                            (types ? (size_t)rows * 2 * sizeof(float) + (size_t)B * sizeof(uint32_t) : 0);
  if (R > 1) {
    e->coef_passes.resize(rows);
    for (int p = 0; p < P; ++p) {
      e->coef_passes[p] = coef[p / R];
      if (p % R != R - 1) e->coef_passes[p].frame = -1;
    }
    e->coef_passes[P] = coef[Tl];
    coef = e->coef_passes.data();
  }
  CK(cudaSetDevice(e->cfg.device));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  cudaStream_t st = e->loop_stream;
  // DL_TIME_CHAIN=1: host-clock breakdown of one call to stderr (adds stream synchronisations: diagnostic only)
  static const bool time_chain = getenv("DL_TIME_CHAIN") != nullptr;
  auto now_ms = [] { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; };
  const double tc0 = time_chain ? now_ms() : 0.0;
  double tc_plan = 0, tc_capture = 0, tc_inst = 0, tc_launch = 0;
  if ((s = ensure_workspace(e, B, N)) != DL_OK) return s;
  if ((size_t)e->coef_cap < coef_bytes) {
    if (e->coef_dev) cudaFree(e->coef_dev);
    e->coef_dev = nullptr;
    CK(cudaMalloc((void**)&e->coef_dev, coef_bytes));
    e->coef_cap = (int)coef_bytes;
  }
  if (e->guide_steps > 0 && e->guide_cap < e->guide_table.size()) {
    if (e->guide_clash) cudaFree(e->guide_clash);
    e->guide_clash = nullptr;
    e->guide_cap = 0;
    CK(cudaMalloc((void**)&e->guide_clash, e->guide_table.size() * sizeof(float)));
    e->guide_cap = e->guide_table.size();
  }
  // order the private loop stream after the caller's stream (the legacy default stream cannot be captured)
  if (user != st) {
    CK(cudaEventRecord(e->ev_in, user));
    CK(cudaStreamWaitEvent(st, e->ev_in, 0));
  }
  CK(cudaMemcpyAsync(e->coef_dev, coef, (size_t)rows * sizeof(dl_step_coef), cudaMemcpyHostToDevice, st));
  if (e->guide_steps > 0)   // the clash-guidance table of this call, ordered on the loop stream like the coefficients
    CK(cudaMemcpyAsync(e->guide_clash, e->guide_table.data(), e->guide_table.size() * sizeof(float), cudaMemcpyHostToDevice,
                       st));
  const float* jump_dev = R > 1 ? e->coef_dev + (size_t)rows * 8 : nullptr;
  if (R > 1)
    CK(cudaMemcpyAsync(const_cast<float*>(jump_dev), e->jump.data(), e->jump.size() * sizeof(float), cudaMemcpyHostToDevice,
                       st));
  const float* ode_dev = ode ? e->coef_dev + (size_t)rows * 8 : nullptr;
  if (ode)
    CK(cudaMemcpyAsync(const_cast<float*>(ode_dev), e->solver_table.data() + (size_t)(T - Tl) * 8,
                       (size_t)rows * 8 * sizeof(float), cudaMemcpyHostToDevice, st));
  const float* fix_dev = fix ? e->coef_dev + (size_t)rows * 8 + (ode ? (size_t)rows * 8 : 0) : nullptr;
  const float* tsc_dev = types ? e->coef_dev + (size_t)rows * 8 + (ode ? (size_t)rows * 8 : 0) + (fix ? (size_t)Tl * 2 : 0)
                               : nullptr;
  const uint32_t* types_dev = types ? reinterpret_cast<const uint32_t*>(tsc_dev + (size_t)rows * 2) : nullptr;
  if (types) {
    // loop row r runs from t = Tl - r: the scalars' row of step t - 1 = T-1-(T-Tl+r-1), or row T where t = T
    std::vector<float> tsc(2 * (size_t)rows);
    for (int r = 0; r < rows; ++r) {
      const int k = T - Tl + r, src = k > 0 ? k - 1 : T;
      tsc[2 * r] = ty.scalars[2 * src]; tsc[2 * r + 1] = ty.scalars[2 * src + 1];
    }
    CK(cudaMemcpyAsync(const_cast<float*>(tsc_dev), tsc.data(), tsc.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(const_cast<uint32_t*>(types_dev), ty.masks, (size_t)B * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  }
  if (fix) {
    CK(cudaMemcpyAsync(const_cast<float*>(fix_dev), fx.scalars + (size_t)(T - Tl) * 2, (size_t)Tl * 2 * sizeof(float),
                       cudaMemcpyHostToDevice, st));
    if (!fx.vetted) {
      // the flags against the masks and the kept types (a recovery round's rows come from a call that passed this)
      // with linker types, also the kept rows' types against their molecules' masks
      int bad[3] = {0, 0, 0};
      CK(cudaMemsetAsync(fx.bad, 0, sizeof(bad), st));
      k_fixed_check<<<(B * N + 255) / 256, 256, 0, st>>>(B * N, 3 + e->cfg.in_node_nf, fx.flags, node_mask, fragment_mask,
                                                        linker_mask, xh, norm[1], norm[2], fx.bad);
      LAUNCH_CHECK();
      e->launches += 1;
      if (types) {
        k_kept_types_check<<<(B * N + 255) / 256, 256, 0, st>>>(B * N, N, 3 + e->cfg.in_node_nf, fx.flags, xh, types_dev,
                                                               norm[1], norm[2], fx.bad + 2);
        LAUNCH_CHECK();
        e->launches += 1;
      }
      CK(cudaMemcpyAsync(bad, fx.bad, sizeof(bad), cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (bad[0] || bad[1] || bad[2]) {
        const int g = (bad[0] ? bad[0] : bad[1] ? bad[1] : bad[2]) - 1;
        set_err("%s: row %d of molecule %d %s", bad[2] && !bad[0] && !bad[1] ? "dl_set_linker_types" : "dl_set_fixed_atoms",
                g % N, g / N,
                bad[0]   ? "is flagged but is not a live linker row (node_mask and linker_mask set, fragment_mask 0)"
                : bad[1] ? "is flagged but its type channels are not a one-hot"
                         : "is kept (dl_set_fixed_atoms) but its type is one its molecule's mask excludes");
        return DL_ERR_INVALID;
      }
    }
  }
  NoiseRng q = rng ? *rng : NoiseRng{};
  // per-molecule start steps: the loop runs on the rows in start-step order, each loop step on those that have started
  RowOrder ro{};
  if (per_row) {
    s = order_rows(e, B, N, Tl, xh, node_mask, fragment_mask, linker_mask, edge_mask, context, per_mol ? rng->seeds : nullptr,
                   fx.flags, st, ro);
    if (s != DL_OK) return s;
    xh = ro.xh; node_mask = ro.node_mask; fragment_mask = ro.fragment_mask; linker_mask = ro.linker_mask;
    edge_mask = ro.edge_mask; context = ro.context;
  }
  const int8_t* fixed = per_row ? ro.fixed : fx.flags;   // in the workspace's row order
  if (per_mol) {
    // the captured step reads the engine's copy: the caller's seeds buffer is free once the call has been enqueued
    if (!per_row)
      CK(cudaMemcpyAsync(e->ws.seeds, rng->seeds, (size_t)B * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    q.seeds = e->ws.seeds;
  }
  CK(cudaMemsetAsync(e->step_ctr, 0, 3 * sizeof(int), st));
  if (nan_flags) CK(cudaMemsetAsync(nan_flags, 0, B * sizeof(int32_t), st));
  const int n = B * N, xd = 3 + e->cfg.in_node_nf;
  // frames that no reverse step is the last writer of stay zero, as torch.zeros in edm.py:143 -- with a start step also
  // every frame whose steps all lie at or above it
  CK(cudaMemsetAsync(chain, 0, (size_t)keep_frames * n * xd * sizeof(float), st));
  if (inpaint && rng) {
    // z_T = COM-free masked noise on every atom (edm.py:565): draw 0 of the device-side stream
    if (per_mol) k_com_free_draws<true><<<dim3(B, 1), 256, 0, st>>>(N, xd, T, q, node_mask, fragment_mask, e->ws.z);
    else k_com_free_draws<false><<<dim3(B, 1), 256, 0, st>>>(N, xd, T, q, node_mask, fragment_mask, e->ws.z);
    LAUNCH_CHECK();
    e->launches += 1;
  } else if (inpaint) {
    // the caller's slab 0 is already masked and projected
    CK(cudaMemcpyAsync(e->ws.z, noise, (size_t)n * xd * sizeof(float), cudaMemcpyDeviceToDevice, st));
  } else if (per_row) {
    if (per_mol) k_init_z_rows<true><<<(n * xd + 255) / 256, 256, 0, st>>>(n, N, xd, xh, fragment_mask, linker_mask, noise, q, ro.alpha, ro.sigma, ro.rs, e->ws.z);
    else k_init_z_rows<false><<<(n * xd + 255) / 256, 256, 0, st>>>(n, N, xd, xh, fragment_mask, linker_mask, noise, q, ro.alpha, ro.sigma, ro.rs, e->ws.z);
    LAUNCH_CHECK();
    e->launches += 1;
  } else if (partial) {
    const float al = e->start_alpha, sg = e->start_sigma;
    if (per_mol) k_init_z_partial<true><<<(n * xd + 255) / 256, 256, 0, st>>>(n, xd, xh, fragment_mask, linker_mask, noise, q, al, sg, e->ws.z);
    else k_init_z_partial<false><<<(n * xd + 255) / 256, 256, 0, st>>>(n, xd, xh, fragment_mask, linker_mask, noise, q, al, sg, e->ws.z);
    LAUNCH_CHECK();
    e->launches += 1;
  } else {
    if (per_mol) k_init_z<true><<<(n * xd + 255) / 256, 256, 0, st>>>(n, xd, xh, fragment_mask, linker_mask, noise, q, e->ws.z);
    else k_init_z<false><<<(n * xd + 255) / 256, 256, 0, st>>>(n, xd, xh, fragment_mask, linker_mask, noise, q, e->ws.z);
    LAUNCH_CHECK();
    e->launches += 1;
  }
  if (fix) {
    // the kept rows start from q(z_t | x) at the call's start: T (the scalars' last row), t0, or each row's own t0
    const float al = partial ? e->start_alpha : fx.scalars[2 * T], sg = partial ? e->start_sigma : fx.scalars[2 * T + 1];
    const float* al_rows = per_row ? ro.alpha : nullptr;
    const float* sg_rows = per_row ? ro.sigma : nullptr;
    const RowStarts rs = per_row ? ro.rs : RowStarts{};
    if (per_mol) k_init_z_fixed<true><<<(n * xd + 255) / 256, 256, 0, st>>>(n, N, xd, xh, fragment_mask, linker_mask, fixed, noise, q, al, sg, al_rows, sg_rows, rs, e->ws.z);
    else k_init_z_fixed<false><<<(n * xd + 255) / 256, 256, 0, st>>>(n, N, xd, xh, fragment_mask, linker_mask, fixed, noise, q, al, sg, al_rows, sg_rows, rs, e->ws.z);
    LAUNCH_CHECK();
    e->launches += 1;
  }
  // inpainting: the dynamics see linker_mask=None (edm.py:632), so every live row gets a coordinate update
  int Bp = per_row ? ro.active[0] : B;   // the rows the current step graph computes
  if ((s = build_forward_plan(e, Bp, N, node_mask, inpaint ? nullptr : linker_mask, edge_mask, st)) != DL_OK) return s;

  if (time_chain) { cudaStreamSynchronize(st); tc_plan = now_ms(); }
  if (e->guide_steps > 0) CK(clash_guide_opt_in());
  FwdIO io;
  io.sampler = true; io.inpaint = inpaint; io.xh0 = xh; io.upd_linker_mask = linker_mask;
  io.node_mask = node_mask; io.linker_mask = inpaint ? nullptr : linker_mask; io.edge_mask = edge_mask;
  io.context = context; io.nan_flags = nan_flags; io.fragment_mask = fragment_mask; io.noise = noise;
  io.rng = q;
  io.chain = chain; io.T = P; io.norm0 = norm[0]; io.norm1 = norm[1]; io.bias1 = norm[2];
  io.rows = per_row ? ro.rs : RowStarts{};
  io.R = R; io.jump = jump_dev; io.ode = ode_dev;
  io.fixed = fixed; io.fix = fix_dev;
  io.types = types_dev; io.tsc = tsc_dev;

  // capture ONE reverse step; the step index lives on the device, so the same graph serves all Tl+1 steps (all P+1 passes
  // with resampling) -- with per-molecule start steps, all steps of one prefix length: the graph is recaptured whenever the
  // prefix grows
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  const int64_t before = e->launches;
  if ((s = capture_step(e, Bp, N, io, st, &graph)) != DL_OK) return s;
  const int64_t per_step = e->launches - before;
  // every exit below releases the captured graph and its executable (destruction is deferred by the runtime until the
  // launched work has finished)
  if (time_chain) tc_capture = now_ms();
  cudaError_t ge = cudaGraphInstantiate(&exec, graph, 0);
  if (time_chain) tc_inst = now_ms();
  if (ge == cudaSuccess) ge = cudaEventRecord(e->ev_t0, st);
  int failed_step = -1;
  int64_t mol_steps = 0, replans = 0;
  for (int r = 0; ge == cudaSuccess && r <= P; ++r) {
    if (per_row && ro.active[r] != Bp) {
      // more rows have started: their plan and step graph, which replaces the executable's (or a new one)
      Bp = ro.active[r];
      ++replans;
      cudaGraph_t next = nullptr;
      s = build_forward_plan(e, Bp, N, node_mask, linker_mask, edge_mask, st);
      if (s == DL_OK) s = capture_step(e, Bp, N, io, st, &next);
      if (s != DL_OK) { cudaGraphExecDestroy(exec); cudaGraphDestroy(graph); return s; }
      cudaGraphDestroy(graph);
      graph = next;
      cudaGraphExecUpdateResultInfo info;
      if (cudaGraphExecUpdate(exec, graph, &info) != cudaSuccess) {
        cudaGetLastError();
        cudaGraphExecDestroy(exec);
        exec = nullptr;
        ge = cudaGraphInstantiate(&exec, graph, 0);
        if (ge != cudaSuccess) break;
      }
    }
    ge = cudaGraphLaunch(exec, st);
    if (ge != cudaSuccess) failed_step = r;
    mol_steps += Bp;
  }
  if (ge == cudaSuccess) ge = cudaEventRecord(e->ev_t1, st);
  if (time_chain) {
    tc_launch = now_ms();
    cudaStreamSynchronize(st);
    const double tc_done = now_ms();
    float loop = 0.f; cudaEventElapsedTime(&loop, e->ev_t0, e->ev_t1);
    fprintf(stderr, "[dl chain] setup+plan %.2f ms | capture %.2f | instantiate %.2f | %d graph launches enqueued in %.2f | wait for the GPU %.2f | device loop %.2f\n",
            tc_plan - tc0, tc_capture - tc_plan, tc_inst - tc_capture, P + 1, tc_launch - tc_inst, tc_done - tc_launch, loop);
  }
  if (ge == cudaSuccess && user != st) {
    ge = cudaEventRecord(e->ev_out, st);
    if (ge == cudaSuccess) ge = cudaStreamWaitEvent(user, e->ev_out, 0);
  }
  if (exec) cudaGraphExecDestroy(exec);
  cudaGraphDestroy(graph);
  if (ge != cudaSuccess) {
    if (failed_step >= 0) set_err("cudaGraphLaunch step %d -> %s", failed_step, cudaGetErrorString(ge));
    else set_err("%s:%d reverse-loop graph -> %s", __FILE__, __LINE__, cudaGetErrorString(ge));
    return DL_ERR_CUDA;
  }
  e->launches = before + per_step * (P + 1) + 2 * replans;
  e->mol_steps = mol_steps;
  return DL_OK;
}

dl_status dl_sample_chain_host(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                               const float* xh, const int8_t* node_mask, const float* fragment_mask,
                               const float* linker_mask, const int8_t* edge_mask, const float* context,
                               const float* noise, const dl_step_coef* coef, const float* norm, float* chain,
                               int32_t* nan_flags) {
  dl_status s = check_shapes(e, B, N);
  if (s == DL_OK) s = check_sampler(e, sampler, T, keep_frames, noise != nullptr, xh, node_mask, fragment_mask, linker_mask,
                                    context, coef, norm, chain);
  if (s != DL_OK) return s;
  CK(cudaSetDevice(e->cfg.device));
  const size_t n = (size_t)B * N, frame_bytes = n * (3 + e->cfg.in_node_nf) * 4;
  const bool fc_em = edge_mask && e->cfg.graph_type == DL_GRAPH_FC;
  const int R = std::max(call_resamplings(e, sampler, T), 1);   // a refused setting fails in dl_sample_chain below
  StageLayout sl;
  const int i_xh = sl.in(xh, frame_bytes), i_nm = sl.in(node_mask, n), i_fm = sl.in(fragment_mask, n * 4),
            i_lm = sl.in(linker_mask, n * 4), i_em = sl.in(fc_em ? edge_mask : nullptr, n * N),
            i_ctx = sl.in(context, n * e->cfg.context_node_nf * 4),
            i_nz = sl.in(noise, sampler_draws(sampler, loop_steps(e, T), R) * frame_bytes),
            i_ch = sl.out(keep_frames * frame_bytes), i_fl = sl.out(B * 4);
  cudaStream_t st = e->loop_stream;
  if ((s = stage_inputs(e->stage, sl, st)) != DL_OK) return s;
  s = dl_sample_chain(e, sampler, B, N, T, keep_frames, sl.at<const float>(i_xh), sl.at<const int8_t>(i_nm),
                      sl.at<const float>(i_fm), sl.at<const float>(i_lm), sl.at<const int8_t>(i_em), sl.at<const float>(i_ctx),
                      sl.at<const float>(i_nz), coef, norm, sl.at<float>(i_ch), sl.at<int32_t>(i_fl), st);
  if (s != DL_OK) return s;
  return stage_results(chain, sl.at<float>(i_ch), keep_frames * frame_bytes, sl.at<int32_t>(i_fl), B, nan_flags, st);
}

uint64_t dl_retry_seed(uint64_t seed, int32_t attempt) { return retry_seed(seed, attempt); }

}  // extern "C"

namespace {

static_assert(CHECK_CONNECTED == DL_CHECK_CONNECTED && CHECK_VALENCE == DL_CHECK_VALENCE && CHECK_CLASH == DL_CHECK_CLASH &&
              CHECK_UNIQUE == DL_CHECK_UNIQUE && CHECK_NOVEL == DL_CHECK_NOVEL && CHECK_RINGS == DL_CHECK_RINGS &&
              CHECK_ANCHORS == DL_CHECK_ANCHORS, "kernels_retry.cuh vs header");

// What is wrong with a caller's dl_molecule_checks for molecules of N rows whose h holds at most max_types type columns, or
// null. The sampler takes every check; dl_molecule_check the bond checks only (the clash check has dl_clash_check,
// DL_CHECK_UNIQUE compares the molecules of one sampling call with each other, which a per-molecule check cannot, and
// DL_CHECK_NOVEL, DL_CHECK_RINGS and DL_CHECK_ANCHORS need a linker_mask).
const char* checks_error(const dl_molecule_checks* ck, int N, int max_types, bool sampler) {
  if (!ck) return "null checks";
  constexpr int hashed = DL_CHECK_UNIQUE | DL_CHECK_NOVEL;
  if (sampler) {
    if (ck->require == 0 || (ck->require & ~(DL_CHECK_CONNECTED | DL_CHECK_VALENCE | DL_CHECK_CLASH | DL_CHECK_UNIQUE |
                                             DL_CHECK_NOVEL | DL_CHECK_RINGS | DL_CHECK_ANCHORS)))
      return "checks->require must be a non-empty OR of DL_CHECK_CONNECTED, DL_CHECK_VALENCE, DL_CHECK_CLASH, "
             "DL_CHECK_UNIQUE, DL_CHECK_NOVEL, DL_CHECK_RINGS and DL_CHECK_ANCHORS";
  } else if (ck->require == 0 || (ck->require & ~(DL_CHECK_CONNECTED | DL_CHECK_VALENCE))) {
    return "checks->require must be DL_CHECK_CONNECTED, DL_CHECK_VALENCE or both (the clash check runs through "
           "dl_clash_check; DL_CHECK_UNIQUE compares the molecules of a dl_sample_chain_retry call with each other, and "
           "dl_molecule_hash gives their hashes; DL_CHECK_NOVEL needs a linker_mask, and its linker hashes are "
           "dl_molecule_hash over node_mask AND linker_mask; DL_CHECK_RINGS runs through dl_ring_check and "
           "DL_CHECK_ANCHORS through dl_anchor_check)";
  }
  if (ck->n_types < 1 || ck->n_types > max_types) return "checks->n_types must be in [1, the width of the atom features]";
  if ((ck->require & (DL_CHECK_CONNECTED | DL_CHECK_VALENCE | hashed | DL_CHECK_RINGS | DL_CHECK_ANCHORS)) && !ck->thr1)
    return "null checks->thr1";
  if ((ck->require & DL_CHECK_VALENCE) && (!ck->thr2 || !ck->thr3 || !ck->max_valence))
    return "DL_CHECK_VALENCE needs checks->thr2, thr3 and max_valence";
  if ((ck->require & DL_CHECK_UNIQUE) && (!ck->thr2 || !ck->thr3)) return "DL_CHECK_UNIQUE needs checks->thr2 and thr3";
  if ((ck->require & DL_CHECK_NOVEL) && (!ck->thr2 || !ck->thr3)) return "DL_CHECK_NOVEL needs checks->thr2 and thr3";
  if (N > CONN_MAX_N) return "the molecule checks take N <= 8192";
  return nullptr;
}

// k_molecule_check over (B, N) molecules with the caller's tables.
CheckArgs check_args(const dl_molecule_checks& ck, const float* xh, int N, int row_stride, const int8_t* node_mask,
                     const float* context, int C, bool drop_pocket, int32_t* passed) {
  CheckArgs ca{};
  ca.xh = xh; ca.N = N; ca.row_stride = row_stride; ca.n_types = ck.n_types;
  ca.thr1 = ck.thr1; ca.thr2 = ck.thr2; ca.thr3 = ck.thr3; ca.max_valence = ck.max_valence;
  ca.node_mask = node_mask; ca.C = C; ca.context = context; ca.drop_pocket = drop_pocket; ca.passed = passed;
  return ca;
}

// ... over frame 0 of a (B, N) chain of this engine's model: ligand rows only on cut-off (pocket) graphs.
CheckArgs check_args(const dl_engine* e, const dl_molecule_checks& ck, const float* chain, int N, const int8_t* node_mask,
                     const float* context, int32_t* passed) {
  return check_args(ck, chain, N, 3 + e->cfg.in_node_nf, node_mask, context, e->cfg.context_node_nf,
                    e->cfg.graph_type != DL_GRAPH_FC, passed);
}

// The anchor flags of a dl_sample_chain_retry call: what dl_set_anchors set since the engine's previous call, or nothing.
struct CallAnchors {
  bool set = false;
  int B = 0, N = 0;
  const int8_t* flags = nullptr;
};

// What is wrong with the checks of a dl_sample_chain_retry call of B molecules, or null.
const char* checked_error(const dl_engine* e, int32_t sampler, int B, int N, const dl_molecule_checks* checks,
                          const CallAnchors& an) {
  const char* why = checks_error(checks, N, e->cfg.in_node_nf, true);
  if (!why && (checks->require & DL_CHECK_CLASH)) {
    if (!checks->clash) why = "DL_CHECK_CLASH needs a clash table (checks->clash)";
    else if (e->cfg.graph_type == DL_GRAPH_FC) why = "DL_CHECK_CLASH needs a pocket: DL_GRAPH_FC graphs have none";
    else if (sampler == DL_SAMPLER_INPAINT) why = "DL_CHECK_CLASH does not take DL_SAMPLER_INPAINT, which re-noises the pocket";
  }
  if (!why && (checks->require & DL_CHECK_RINGS) && !e->ring_set)
    why = "DL_CHECK_RINGS in checks->require needs the allowed ring sizes: call dl_set_ring_sizes first";
  if (!why && (checks->require & DL_CHECK_ANCHORS)) {
    if (!an.set) why = "DL_CHECK_ANCHORS in checks->require needs the anchor flags: call dl_set_anchors before every call";
    else if (an.B != B || an.N != N) why = "DL_CHECK_ANCHORS: dl_set_anchors was called with another B or N";
  }
  return why;
}

// What is wrong with a dl_size_redraw for B molecules of N rows, or null. Copies the size table and n_frag to the host
// through `st` (the call blocks anyway) to check that every redrawn template fits N rows.
const char* redraw_error(int32_t sampler, int B, int N, const dl_size_redraw* rz, cudaStream_t st) {
  if (sampler == DL_SAMPLER_INPAINT) return "DL_SAMPLER_INPAINT samples every atom of the batch: it has no linker size to redraw";
  if (rz->C < 1 || rz->logits_row_stride < rz->C) return "redraw->C must be >= 1 and redraw->logits_row_stride >= C";
  if (!rz->logits || !rz->sizes || !rz->n_frag || !rz->linker_x) return "null redraw->logits, sizes, n_frag or linker_x";
  if (B < 1 || N < 1) return "B and N must be >= 1";
  std::vector<int32_t> sizes(rz->C), n_frag(B);
  if (cudaMemcpyAsync(sizes.data(), rz->sizes, sizes.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaMemcpyAsync(n_frag.data(), rz->n_frag, n_frag.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess) {
    cudaGetLastError();
    return "redraw->sizes and n_frag must be DEVICE buffers";
  }
  const int32_t max_size = *std::max_element(sizes.begin(), sizes.end());
  if (*std::min_element(sizes.begin(), sizes.end()) < 0) return "redraw->sizes must be >= 0";
  for (int b = 0; b < B; ++b) {
    if (n_frag[b] < 0) return "redraw->n_frag must be >= 0";
    if ((int64_t)n_frag[b] + max_size > N) return "N < n_frag[b] + max(sizes) for some b: pad the batch to its capacity";
  }
  return nullptr;
}

// Whether p is device memory of `device` or managed memory, by cudaPointerGetAttributes: what a kernel on that device may
// read. Host, unregistered and unknown pointers are not.
bool device_readable(const void* p, int device) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeManaged || (at.type == cudaMemoryTypeDevice && at.device == device);
}

// What is wrong with the hash sets of a dl_sample_chain_retry_sets call whose checks require `require`, or null. Checks
// through `st` (the call blocks anyway) that every set in use is ascending.
const char* sets_error(dl_engine* e, int require, const dl_hash_sets* hs, cudaStream_t st) {
  if (hs->n_known < 0 || hs->n_seen < 0) return "sets->n_known and n_seen must be >= 0";
  const bool known = (require & DL_CHECK_NOVEL) && hs->n_known > 0, seen = (require & DL_CHECK_UNIQUE) && hs->n_seen > 0;
  if ((known && !hs->known) || (seen && !hs->seen)) return "null sets->known or seen with a positive count";
  if (!known && !seen) return nullptr;
  if ((known && !device_readable(hs->known, e->cfg.device)) || (seen && !device_readable(hs->seen, e->cfg.device)))
    return "sets->known and seen must be device (or managed) memory of the engine's device";
  if (cudaSetDevice(e->cfg.device) != cudaSuccess) return "cudaSetDevice failed";
  StageLayout sl;
  const int i_bad = sl.out(2 * sizeof(int32_t));
  if (stage_inputs(e->sub_rows, sl, st) != DL_OK) return "could not allocate the set check's flags";
  int32_t* bad = sl.at<int32_t>(i_bad);
  int32_t h_bad[2] = {0, 0};
  bool ok = cudaMemsetAsync(bad, 0, 2 * sizeof(int32_t), st) == cudaSuccess;
  const std::pair<const uint64_t*, int64_t> sets[2] = {{known ? hs->known : nullptr, hs->n_known},
                                                       {seen ? hs->seen : nullptr, hs->n_seen}};
  for (int k = 0; k < 2 && ok; ++k) {
    if (!sets[k].first || sets[k].second < 2) continue;
    const int64_t blocks = std::min<int64_t>((sets[k].second + 255) / 256, 1024);
    k_sorted_check<<<(int)blocks, 256, 0, st>>>(reinterpret_cast<const unsigned long long*>(sets[k].first), sets[k].second,
                                                bad + k);
    ok = cudaGetLastError() == cudaSuccess;
    e->launches += 1;
  }
  ok = ok && cudaMemcpyAsync(h_bad, bad, sizeof(h_bad), cudaMemcpyDeviceToHost, st) == cudaSuccess &&
       cudaStreamSynchronize(st) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    return "the check of sets->known and seen failed";
  }
  if (h_bad[0]) return "sets->known is not in ascending unsigned order";
  if (h_bad[1]) return "sets->seen is not in ascending unsigned order";
  return nullptr;
}

// dl_sample_chain_retry, and with `ck` its molecule checks, whose verdicts go to `passed`: a row then fails if its NaN
// flag is set or a required bit is missing, and a resampled row replaces the caller's unless the caller's row is finite and
// the new one diverged. `hs` (or null) holds the known set of DL_CHECK_NOVEL and the seen set of DL_CHECK_UNIQUE;
// `linker_hash` (or null) receives every returned row's linker hash with DL_CHECK_NOVEL. `anchors` (B, N), read with
// DL_CHECK_ANCHORS only, are the anchor flags, which k_anchor_check reads right after the check launch. `fx` are the call's
// fixed atoms: every round gathers its rows' flags and keeps them. `ty` are the call's linker types: every round takes its
// rows' masks.
dl_status seeded_retry(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames, const float* xh,
                       const int8_t* node_mask, const float* fragment_mask, const float* linker_mask, const int8_t* edge_mask,
                       const float* context, const uint64_t* seeds, const dl_step_coef* coef, const float* norm, float* chain,
                       int32_t* nan_flags, int32_t max_retries, uint64_t* seeds_used, int32_t* attempts,
                       const dl_molecule_checks* ck, const dl_hash_sets* hs, int32_t* passed, uint64_t* linker_hash,
                       const dl_size_redraw* rz, int32_t* sizes_used, const int8_t* anchors, const CallFixed& fx,
                       const CallTypes& ty, void* stream) {
  e->retry_ms = 0.f;
  e->ring_B = 0;
  dl_status s = sample_seeded(e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask, linker_mask, edge_mask, context,
                              seeds, coef, norm, chain, nan_flags, stream, fx, ty);
  if (s != DL_OK) return s;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CK(cudaMemcpyAsync(seeds_used, seeds, (size_t)B * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemsetAsync(attempts, 0, (size_t)B * sizeof(int32_t), st));
  const int require = ck ? ck->require : 0;
  const bool unique = (require & DL_CHECK_UNIQUE) != 0;
  const bool seen = unique && hs && hs->n_seen > 0;        // the verdict's seen set
  const SeenArgs sn{seen ? reinterpret_cast<const unsigned long long*>(hs->seen) : nullptr, seen ? hs->n_seen : 0};
  const bool known = (require & DL_CHECK_NOVEL) && hs && hs->n_known > 0;
  const unsigned long long* kn = known ? reinterpret_cast<const unsigned long long*>(hs->known) : nullptr;
  const long long n_known = known ? hs->n_known : 0;
  unsigned long long* lh = (require & DL_CHECK_NOVEL) ? reinterpret_cast<unsigned long long*>(linker_hash) : nullptr;
  std::vector<int32_t> flags(B), pass(B, require);
  unsigned long long* hash = nullptr;                      // DL_CHECK_UNIQUE: the full batch's graph hashes
  if (unique) {
    StageLayout hl;
    hl.out((size_t)B * sizeof(uint64_t));
    if ((s = stage_inputs(e->hashes, hl, st)) != DL_OK) return s;
    hash = reinterpret_cast<unsigned long long*>(e->hashes.buf);
  }
  const bool rings = (require & DL_CHECK_RINGS) != 0;
  unsigned long long* ring_masks = nullptr;                // DL_CHECK_RINGS: every returned row's mask (dl_last_ring_sizes)
  if (rings) {
    StageLayout rl;
    rl.out((size_t)B * sizeof(uint64_t));
    if ((s = stage_inputs(e->ring_masks, rl, st)) != DL_OK) return s;
    ring_masks = reinterpret_cast<unsigned long long*>(e->ring_masks.buf);
  }
  // DL_CHECK_ANCHORS has a launch of its own after the check launch (which takes the other bits, if any), before the
  // uniqueness verdict, whose eligible candidates need every other required bit
  const int mol = require & ~DL_CHECK_ANCHORS;
  const bool anchored = (require & DL_CHECK_ANCHORS) != 0;
  if (ck) {
    const ClashArgs cl{linker_mask, ck->clash, nullptr};   // the clash check's linker rows and table
    const CheckArgs ca = check_args(e, *ck, chain, N, node_mask, context, passed);
    if (mol) {
      CK(launch_molecule_check(mol, ca, cl, HashArgs{hash, 0}, B, st, NovelArgs{linker_mask, kn, n_known, lh},
                               e->ring_allowed, ring_masks));
      e->launches += 1;
    }
    if (anchored) {
      CK(launch_anchor_check(ca, AnchorArgs{linker_mask, anchors, nullptr, mol != 0}, B, st));
      e->launches += 1;
    }
    if (unique) {                                          // every row is a candidate; the only keepers are the seen set
      UniqueArgs u{};
      u.B = B; u.require = require; u.hash = hash; u.flags = nan_flags; u.passed = passed;
      if (seen) k_unique_verdict<<<(B + 255) / 256, 256, 0, st>>>(u, sn);
      else k_unique_verdict<<<(B + 255) / 256, 256, 0, st>>>(u);
      LAUNCH_CHECK();
      e->launches += 1;
    }
    CK(cudaMemcpyAsync(pass.data(), passed, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  }
  CK(cudaMemcpyAsync(flags.data(), nan_flags, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  // cut-off graphs never read edge_mask (the reference's batch-id vector is implied by the layout): the sub-batch gets none
  const bool fc_em = edge_mask && e->cfg.graph_type == DL_GRAPH_FC;
  const int xd = 3 + e->cfg.in_node_nf, C = e->cfg.context_node_nf;
  for (int a = 1; a <= max_retries; ++a) {
    std::vector<int32_t> rows;
    for (int b = 0; b < B; ++b) if (flags[b] != 0 || pass[b] != require) rows.push_back(b);
    if (rows.empty()) break;
    const int Bs = (int)rows.size();
    const size_t n = (size_t)Bs * N;
    StageLayout sl;
    const int i_rows = sl.in(rows.data(), (size_t)Bs * sizeof(int32_t)), i_xh = sl.out(n * xd * 4), i_nm = sl.out(n),
              i_fm = sl.out(n * 4), i_lm = sl.out(n * 4), i_em = sl.add(nullptr, n * N, fc_em),
              i_ctx = sl.add(nullptr, n * C * 4, context != nullptr && C > 0), i_sd = sl.out((size_t)Bs * 8),
              i_ch = sl.out((size_t)keep_frames * n * xd * 4), i_fl = sl.out((size_t)Bs * 4),
              i_ps = sl.add(nullptr, (size_t)Bs * 4, ck != nullptr), i_tk = sl.add(nullptr, (size_t)Bs * 4, ck != nullptr),
              i_sz = sl.add(nullptr, (size_t)Bs * 4, rz != nullptr), i_sh = sl.add(nullptr, (size_t)Bs * 8, unique),
              i_fx = sl.add(nullptr, n, fx.flags != nullptr);
    if ((s = stage_inputs(e->sub_rows, sl, st)) != DL_OK) return s;   // the row list goes to the device once per round
    CK(cudaEventRecord(e->ev_g0, st));
    RowGatherArgs ga{};
    ga.rows = sl.at<const int>(i_rows); ga.N = N; ga.xd = xd; ga.C = C; ga.attempt = a;
    ga.xh = xh; ga.fragment_mask = fragment_mask; ga.linker_mask = linker_mask; ga.context = sl.at<float>(i_ctx) ? context : nullptr;
    ga.node_mask = node_mask; ga.edge_mask = fc_em ? edge_mask : nullptr;
    ga.seeds = reinterpret_cast<const unsigned long long*>(seeds);
    ga.s_xh = sl.at<float>(i_xh); ga.s_fragment_mask = sl.at<float>(i_fm); ga.s_linker_mask = sl.at<float>(i_lm);
    ga.s_context = sl.at<float>(i_ctx); ga.s_node_mask = sl.at<int8_t>(i_nm); ga.s_edge_mask = sl.at<int8_t>(i_em);
    ga.s_seeds = sl.at<unsigned long long>(i_sd);
    const RowFixedArgs fa{fx.flags, sl.at<int8_t>(i_fx)};
    const RowSizeArgs za{sl.at<int32_t>(i_sz), sizes_used};
    if (rz) {
      const RowResizeArgs ra{SizeDrawArgs{rz->C, rz->logits_row_stride, rz->logits, rz->sizes}, rz->n_frag, rz->linker_x,
                             sl.at<int32_t>(i_sz)};
      k_gather_rows<true><<<Bs, 256, 0, st>>>(ga, ra);
    } else if (fx.flags) {
      k_gather_rows<false><<<Bs, 256, 0, st>>>(ga, fa);
    } else {
      k_gather_rows<false><<<Bs, 256, 0, st>>>(ga);
    }
    LAUNCH_CHECK();
    e->launches += 1;
    // with per-molecule start steps, the sub-batch carries each failing row's step and scalars
    std::vector<int32_t> t0_all;
    std::vector<float> alpha_all, sigma_all;
    const bool per_row = !e->starts_t0.empty();
    if (per_row) {
      t0_all.swap(e->starts_t0); alpha_all.swap(e->starts_alpha); sigma_all.swap(e->starts_sigma);
      for (int b : rows) {
        e->starts_t0.push_back(t0_all[b]); e->starts_alpha.push_back(alpha_all[b]); e->starts_sigma.push_back(sigma_all[b]);
      }
    }
    {
      SubBatchScope sub(e);
      CallFixed sub_fx;                                    // the round's rows keep their fixed atoms
      if (fx.flags) {
        sub_fx = fx;
        sub_fx.flags = fa.s_fixed; sub_fx.B = Bs; sub_fx.vetted = true;
      }
      std::vector<uint32_t> sub_masks;                     // ... and their linker types
      CallTypes sub_ty;
      if (ty.masks) {
        for (int b : rows) sub_masks.push_back(ty.masks[b]);
        sub_ty = ty;
        sub_ty.masks = sub_masks.data(); sub_ty.B = Bs;
      }
      s = sample_seeded(e, sampler, Bs, N, T, keep_frames, ga.s_xh, ga.s_node_mask, ga.s_fragment_mask, ga.s_linker_mask,
                        ga.s_edge_mask, ga.s_context, reinterpret_cast<const uint64_t*>(ga.s_seeds), coef, norm,
                        sl.at<float>(i_ch), sl.at<int32_t>(i_fl), stream, sub_fx, sub_ty);
    }
    if (per_row) { e->starts_t0.swap(t0_all); e->starts_alpha.swap(alpha_all); e->starts_sigma.swap(sigma_all); }
    if (s != DL_OK) return s;
    RowScatterArgs sa{};
    sa.rows = ga.rows; sa.B = B; sa.Bs = Bs; sa.N = N; sa.xd = xd; sa.attempt = a;
    sa.s_chain = sl.at<float>(i_ch); sa.s_flags = sl.at<int32_t>(i_fl); sa.s_seeds = ga.s_seeds;
    sa.chain = chain; sa.flags = nan_flags; sa.seeds_used = reinterpret_cast<unsigned long long*>(seeds_used);
    sa.attempts = attempts;
    if (ck) {
      CheckArgs ca = check_args(e, *ck, sa.s_chain, N, ga.s_node_mask, ga.s_context, sl.at<int32_t>(i_ps));
      ca.rows = ga.rows; ca.flags = nan_flags; ca.s_flags = sa.s_flags; ca.take = sl.at<int32_t>(i_tk);
      const HashArgs ha{sl.at<unsigned long long>(i_sh), 0};
      if (mol) {
        CK(launch_molecule_check(mol, ca, ClashArgs{ga.s_linker_mask, ck->clash, nullptr}, ha, Bs, st,
                                 NovelArgs{ga.s_linker_mask, kn, n_known, lh}, e->ring_allowed, ring_masks));
        e->launches += 1;
      }
      if (anchored) {                                      // the caller's row rows[i], row for row
        CK(launch_anchor_check(ca, AnchorArgs{ga.s_linker_mask, anchors, nullptr, mol != 0}, Bs, st));
        e->launches += 1;
      }
      sa.take = ca.take; sa.s_passed = ca.passed; sa.passed = passed;
      if (rz) k_scatter_rows<true><<<dim3(Bs, keep_frames), 256, 0, st>>>(sa, za);
      else k_scatter_rows<true><<<dim3(Bs, keep_frames), 256, 0, st>>>(sa);
    } else if (rz) {
      k_scatter_rows<false><<<dim3(Bs, keep_frames), 256, 0, st>>>(sa, za);
    } else {
      k_scatter_rows<false><<<dim3(Bs, keep_frames), 256, 0, st>>>(sa);
    }
    LAUNCH_CHECK();
    e->launches += 1;
    if (unique) {                                          // the round's rows against the keepers and each other
      UniqueArgs u{};
      u.B = B; u.Bs = Bs; u.require = require; u.hash = hash; u.flags = nan_flags; u.passed = passed;
      u.rows = ga.rows; u.take = sa.take; u.s_hash = sl.at<unsigned long long>(i_sh);
      if (seen) k_unique_verdict<<<(Bs + 255) / 256, 256, 0, st>>>(u, sn);
      else k_unique_verdict<<<(Bs + 255) / 256, 256, 0, st>>>(u);
      LAUNCH_CHECK();
      e->launches += 1;
    }
    CK(cudaEventRecord(e->ev_g1, st));
    std::vector<int32_t> sub_flags(Bs), sub_pass(Bs, require), take(Bs, 1);
    CK(cudaMemcpyAsync(sub_flags.data(), sa.s_flags, (size_t)Bs * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (ck) {
      CK(cudaMemcpyAsync(sub_pass.data(), sa.s_passed, (size_t)Bs * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(take.data(), sa.take, (size_t)Bs * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    }
    // the verdict may change the bit of rows that were not taken too: read every row's verdict
    if (unique) CK(cudaMemcpyAsync(pass.data(), passed, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e->ev_g0, e->ev_g1));
    e->retry_ms += ms;
    for (int i = 0; i < Bs; ++i)
      if (take[i]) { flags[rows[i]] = sub_flags[i]; if (!unique) pass[rows[i]] = sub_pass[i]; }
  }
  if (rings) e->ring_B = B;
  for (int b = 0; b < B; ++b) if (flags[b] != 0) return DL_NAN_DETECTED;
  return DL_OK;
}

// The argument checks of dl_sample_chain_retry(_sets) `name`, then seeded_retry.
dl_status retry_entry(const char* name, dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                      const float* xh, const int8_t* node_mask, const float* fragment_mask, const float* linker_mask,
                      const int8_t* edge_mask, const float* context, const uint64_t* seeds, const dl_step_coef* coef,
                      const float* norm, float* chain, int32_t* nan_flags, int32_t max_retries, uint64_t* seeds_used,
                      int32_t* attempts, const dl_molecule_checks* checks, const dl_hash_sets* sets, int32_t* passed,
                      uint64_t* linker_hash, const dl_size_redraw* redraw, int32_t* sizes_used, void* stream) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  CallAnchors an;                                          // read and cleared by every call, whatever it requires
  an.set = e->anchors_set; an.B = e->anchors_B; an.N = e->anchors_N;
  an.flags = reinterpret_cast<const int8_t*>(e->anchors.buf);
  e->anchors_set = false;
  const CallFixed fx = take_fixed(e);                      // likewise
  const CallTypes ty = take_types(e);                      // likewise
  if (max_retries < 0) { set_err("max_retries must be >= 0 (got %d)", max_retries); return DL_ERR_INVALID; }
  if (!nan_flags || !seeds_used || !attempts || (checks && !passed) || (redraw && !sizes_used)) {
    set_err("%s: null argument (nan_flags, seeds_used, attempts, passed with checks or sizes_used with redraw)", name);
    return DL_ERR_INVALID;
  }
  const char* why = checks ? checked_error(e, sampler, B, N, checks, an) : nullptr;
  if (!why && linker_hash && !(checks && (checks->require & DL_CHECK_NOVEL)))
    why = "linker_hash needs checks with DL_CHECK_NOVEL";
  if (!why && sets && !checks) why = "sets need checks: the known set is read with DL_CHECK_NOVEL, the seen set with "
                                     "DL_CHECK_UNIQUE";
  if (!why && redraw && !e->starts_t0.empty())
    why = "a size redraw takes no start steps: partial diffusion varies the batch's own linker, whose size is given";
  if (!why && redraw && fx.flags)
    why = "a size redraw takes no fixed atoms (dl_set_fixed_atoms): it rebuilds the linker rows at new sizes";
  if (!why && redraw) {
    if (cudaSetDevice(e->cfg.device) != cudaSuccess) why = "cudaSetDevice failed";
    else why = redraw_error(sampler, B, N, redraw, reinterpret_cast<cudaStream_t>(stream));
  }
  if (!why && sets) why = sets_error(e, checks->require, sets, reinterpret_cast<cudaStream_t>(stream));
  if (why) {
    set_err("%s: %s", name, why);
    return DL_ERR_INVALID;
  }
  return seeded_retry(e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask, linker_mask, edge_mask, context, seeds,
                      coef, norm, chain, nan_flags, max_retries, seeds_used, attempts, checks, sets, passed, linker_hash,
                      redraw, sizes_used, an.flags, fx, ty, stream);
}

}  // namespace

extern "C" {

dl_status dl_sample_chain_retry(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                const float* xh, const int8_t* node_mask, const float* fragment_mask, const float* linker_mask,
                                const int8_t* edge_mask, const float* context, const uint64_t* seeds, const dl_step_coef* coef,
                                const float* norm, float* chain, int32_t* nan_flags, int32_t max_retries, uint64_t* seeds_used,
                                int32_t* attempts, const dl_molecule_checks* checks, int32_t* passed,
                                const dl_size_redraw* redraw, int32_t* sizes_used, void* stream) {
  return retry_entry("dl_sample_chain_retry", e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask, linker_mask,
                     edge_mask, context, seeds, coef, norm, chain, nan_flags, max_retries, seeds_used, attempts, checks,
                     nullptr, passed, nullptr, redraw, sizes_used, stream);
}

dl_status dl_sample_chain_retry_sets(dl_engine* e, int32_t sampler, int32_t B, int32_t N, int32_t T, int32_t keep_frames,
                                     const float* xh, const int8_t* node_mask, const float* fragment_mask,
                                     const float* linker_mask, const int8_t* edge_mask, const float* context,
                                     const uint64_t* seeds, const dl_step_coef* coef, const float* norm, float* chain,
                                     int32_t* nan_flags, int32_t max_retries, uint64_t* seeds_used, int32_t* attempts,
                                     const dl_molecule_checks* checks, const dl_hash_sets* sets, int32_t* passed,
                                     uint64_t* linker_hashes, const dl_size_redraw* redraw, int32_t* sizes_used,
                                     void* stream) {
  return retry_entry("dl_sample_chain_retry_sets", e, sampler, B, N, T, keep_frames, xh, node_mask, fragment_mask,
                     linker_mask, edge_mask, context, seeds, coef, norm, chain, nan_flags, max_retries, seeds_used, attempts,
                     checks, sets, passed, linker_hashes, redraw, sizes_used, stream);
}

dl_status dl_size_draw(int32_t B, int32_t C, const float* logits, int32_t logits_row_stride, const int32_t* sizes,
                       const uint64_t* seeds, int32_t attempt, int32_t* out_sizes, void* stream) {
  const char* why = nullptr;
  if (B <= 0 || C <= 0) why = "B and C must be >= 1";
  else if (logits_row_stride < C) why = "logits_row_stride must be >= C";
  else if (!logits || !sizes || !seeds || !out_sizes) why = "null argument";
  if (why) { set_err("dl_size_draw: %s", why); return DL_ERR_INVALID; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  k_size_draw<<<(B + 7) / 8, 256, 0, st>>>(SizeDrawArgs{C, logits_row_stride, logits, sizes}, B,
                                           reinterpret_cast<const unsigned long long*>(seeds), attempt, out_sizes);
  CK(cudaGetLastError());
  return DL_OK;
}

double dl_size_uniform(uint64_t seed) { return size_uniform(seed); }

dl_status dl_molecule_check(int32_t B, int32_t N, const dl_molecule_checks* checks, const float* xh, int32_t xh_row_stride,
                            const int8_t* node_mask, const float* context, int32_t context_nf, int32_t drop_pocket,
                            int32_t* passed, int32_t* valence, void* stream) {
  const char* why = checks_error(checks, N, xh_row_stride - 3, false);
  if (!why && (B <= 0 || N <= 0 || !xh || !node_mask || !passed || (drop_pocket && (!context || context_nf < 1))))
    why = "invalid argument";
  if (!why && valence && !(checks->require & DL_CHECK_VALENCE)) why = "valence needs DL_CHECK_VALENCE";
  if (why) { set_err("dl_molecule_check: %s", why); return DL_ERR_INVALID; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CheckArgs ca = check_args(*checks, xh, N, xh_row_stride, node_mask, context, context_nf, drop_pocket != 0, passed);
  ca.valence = valence;
  if (valence) CK(cudaMemsetAsync(valence, 0, (size_t)B * N * sizeof(int32_t), st));   // the rows that are not checked
  CK(launch_molecule_check(checks->require, ca, ClashArgs{}, HashArgs{}, B, st));
  return DL_OK;
}

dl_status dl_molecule_hash(int32_t B, int32_t N, const dl_molecule_checks* checks, const float* xh, int32_t xh_row_stride,
                           const int8_t* node_mask, const float* context, int32_t context_nf, int32_t drop_pocket,
                           uint64_t* hash, void* stream) {
  const char* why = nullptr;
  if (!checks) why = "null checks";
  else if (B <= 0 || N <= 0) why = "B and N must be >= 1";
  else if (N > CONN_MAX_N) why = "the molecule checks take N <= 8192";
  else if (checks->n_types < 1 || checks->n_types > xh_row_stride - 3) why = "checks->n_types must be in [1, xh_row_stride - 3]";
  else if (!checks->thr1 || !checks->thr2 || !checks->thr3) why = "the hash needs checks->thr1, thr2 and thr3";
  else if (!xh || !node_mask || !hash || (drop_pocket && (!context || context_nf < 1))) why = "invalid argument";
  if (why) { set_err("dl_molecule_hash: %s", why); return DL_ERR_INVALID; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CheckArgs ca = check_args(*checks, xh, N, xh_row_stride, node_mask, context, context_nf, drop_pocket != 0, nullptr);
  CK(launch_molecule_check(CHECK_UNIQUE, ca, ClashArgs{}, HashArgs{reinterpret_cast<unsigned long long*>(hash), 0}, B, st));
  return DL_OK;
}

dl_status dl_novel_check(int32_t B, int32_t N, const dl_molecule_checks* checks, const dl_hash_sets* sets, const float* xh,
                         int32_t xh_row_stride, const int8_t* node_mask, const float* linker_mask, const float* context,
                         int32_t context_nf, int32_t drop_pocket, int32_t* passed, uint64_t* linker_hash, uint64_t* hash,
                         void* stream) {
  const char* why = checks_error(checks, N, xh_row_stride - 3, true);
  const int require = checks ? checks->require : 0;
  int dev = 0;
  if (!why && (require & (DL_CHECK_RINGS | DL_CHECK_ANCHORS)))
    why = "checks->require must be an OR of DL_CHECK_NOVEL and the bits below (DL_CHECK_RINGS runs through dl_ring_check, "
          "DL_CHECK_ANCHORS through dl_anchor_check)";
  else if (!why && !(require & DL_CHECK_NOVEL)) why = "checks->require must include DL_CHECK_NOVEL";
  else if (!why && (B <= 0 || N <= 0 || !xh || !node_mask || !linker_mask || !passed ||
                    (drop_pocket && (!context || context_nf < 1))))
    why = "invalid argument";
  else if (!why && (require & DL_CHECK_UNIQUE) && !hash) why = "DL_CHECK_UNIQUE needs `hash`";
  else if (!why && (require & DL_CHECK_CLASH) && (!checks->clash || !drop_pocket))
    why = "DL_CHECK_CLASH needs checks->clash and drop_pocket (the pocket rows)";
  else if (!why && sets && sets->n_known < 0) why = "sets->n_known must be >= 0";
  else if (!why && sets && sets->n_known > 0 &&
           (!sets->known || cudaGetDevice(&dev) != cudaSuccess || !device_readable(sets->known, dev)))
    why = "sets->known must be device (or managed) memory of the current device";
  if (why) { set_err("dl_novel_check: %s", why); return DL_ERR_INVALID; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CheckArgs ca = check_args(*checks, xh, N, xh_row_stride, node_mask, context, context_nf, drop_pocket != 0, passed);
  const bool known = sets && sets->n_known > 0;
  const NovelArgs nv{linker_mask, known ? reinterpret_cast<const unsigned long long*>(sets->known) : nullptr,
                     known ? sets->n_known : 0, reinterpret_cast<unsigned long long*>(linker_hash)};
  CK(launch_molecule_check(require, ca, ClashArgs{linker_mask, checks->clash, nullptr},
                           HashArgs{reinterpret_cast<unsigned long long*>(hash), 0}, B, st, nv));
  return DL_OK;
}

dl_status dl_clash_check(int32_t B, int32_t N, int32_t n_types, const float* clash, const float* xh, int32_t xh_row_stride,
                         const int8_t* node_mask, const float* linker_mask, const float* context, int32_t context_nf,
                         int32_t* passed, int32_t* clashes, void* stream) {
  const char* why = nullptr;
  if (B <= 0 || N <= 0) why = "B and N must be >= 1";
  else if (N > CONN_MAX_N) why = "the molecule checks take N <= 8192";
  else if (n_types < 1 || n_types > xh_row_stride - 3) why = "n_types must be in [1, xh_row_stride - 3]";
  else if (!clash) why = "null clash table";
  else if (!xh || !node_mask || !linker_mask || !context || context_nf < 1 || !passed) why = "invalid argument";
  if (why) { set_err("dl_clash_check: %s", why); return DL_ERR_INVALID; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CheckArgs ca{};
  ca.xh = xh; ca.N = N; ca.row_stride = xh_row_stride; ca.n_types = n_types;
  ca.node_mask = node_mask; ca.C = context_nf; ca.context = context; ca.drop_pocket = 1; ca.passed = passed;
  if (clashes) CK(cudaMemsetAsync(clashes, 0, (size_t)B * N * sizeof(int32_t), st));   // the rows that are not linker atoms
  CK(launch_molecule_check(CHECK_CLASH, ca, ClashArgs{linker_mask, clash, clashes}, HashArgs{}, B, st));
  return DL_OK;
}

dl_status dl_clash_guide(int32_t B, int32_t N, int32_t n_types, const float* clash, float scale, float* xh,
                         int32_t xh_row_stride, const int8_t* node_mask, const float* linker_mask, const float* context,
                         int32_t context_nf, void* stream) {
  const char* why = nullptr;
  if (B <= 0 || N <= 0) why = "B and N must be >= 1";
  else if (N > CONN_MAX_N) why = "it takes N <= 8192";
  else if (n_types < 1 || n_types > xh_row_stride - 3) why = "n_types must be in [1, xh_row_stride - 3]";
  else if (!clash) why = "null clash table";
  else if (!std::isfinite(scale) || scale < 0.f) why = "scale must be finite and >= 0";
  else if (!xh || !node_mask || !linker_mask || !context || context_nf < 1) why = "invalid argument";
  if (why) { set_err("dl_clash_guide: %s", why); return DL_ERR_INVALID; }
  if (scale == 0.f) return DL_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CK(clash_guide_opt_in());
  GuideArgs ga{};
  ga.xh = xh; ga.N = N; ga.row_stride = xh_row_stride; ga.n_types = n_types; ga.C = context_nf;
  ga.scale = scale; ga.clash = clash; ga.node_mask = node_mask; ga.linker_mask = linker_mask; ga.context = context;
  CK(launch_clash_guide(ga, B, st));
  return DL_OK;
}

dl_status dl_ring_check(int32_t B, int32_t N, int32_t n_types, const float* thr1, const float* xh, int32_t xh_row_stride,
                        const int8_t* node_mask, const float* linker_mask, const float* context, int32_t context_nf,
                        int32_t drop_pocket, uint64_t allowed, int32_t* passed, uint64_t* ring_sizes, void* stream) {
  const char* why = nullptr;
  if (B <= 0 || N <= 0) why = "B and N must be >= 1";
  else if (N > CONN_MAX_N) why = "the molecule checks take N <= 8192";
  else if (n_types < 1 || n_types > xh_row_stride - 3) why = "n_types must be in [1, xh_row_stride - 3]";
  else if (allowed & 7u) why = "bits 0-2 of allowed must be clear (a ring has at least 3 atoms)";
  else if (!thr1 || !xh || !node_mask || !linker_mask || !passed || (drop_pocket && (!context || context_nf < 1)))
    why = "invalid argument";
  if (why) { set_err("dl_ring_check: %s", why); return DL_ERR_INVALID; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CheckArgs ca{};
  ca.xh = xh; ca.N = N; ca.row_stride = xh_row_stride; ca.n_types = n_types; ca.thr1 = thr1;
  ca.node_mask = node_mask; ca.C = context_nf; ca.context = context; ca.drop_pocket = drop_pocket != 0; ca.passed = passed;
  CK(launch_molecule_check(CHECK_RINGS, ca, ClashArgs{}, HashArgs{}, B, st, NovelArgs{linker_mask, nullptr, 0, nullptr},
                           allowed, reinterpret_cast<unsigned long long*>(ring_sizes)));
  return DL_OK;
}

dl_status dl_anchor_check(int32_t B, int32_t N, int32_t n_types, const float* thr1, const float* xh, int32_t xh_row_stride,
                          const int8_t* node_mask, const float* linker_mask, const int8_t* anchors, const float* context,
                          int32_t context_nf, int32_t drop_pocket, int32_t* passed, int32_t* attachments, void* stream) {
  const char* why = nullptr;
  if (B <= 0 || N <= 0) why = "B and N must be >= 1";
  else if (N > CONN_MAX_N) why = "the molecule checks take N <= 8192";
  else if (n_types < 1 || n_types > xh_row_stride - 3) why = "n_types must be in [1, xh_row_stride - 3]";
  else if (!thr1 || !xh || !node_mask || !linker_mask || !anchors || !passed ||
           (drop_pocket && (!context || context_nf < 1)))
    why = "invalid argument";
  if (why) { set_err("dl_anchor_check: %s", why); return DL_ERR_INVALID; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CheckArgs ca{};
  ca.xh = xh; ca.N = N; ca.row_stride = xh_row_stride; ca.n_types = n_types; ca.thr1 = thr1;
  ca.node_mask = node_mask; ca.C = context_nf; ca.context = context; ca.drop_pocket = drop_pocket != 0; ca.passed = passed;
  CK(launch_anchor_check(ca, AnchorArgs{linker_mask, anchors, attachments, 0}, B, st));
  return DL_OK;
}

dl_status dl_last_ring_sizes(dl_engine* e, int32_t B, uint64_t* out, void* stream) {
  const char* why = nullptr;
  if (!e || !out) why = "null engine or out";
  else if (e->ring_B == 0) why = "the last dl_sample_chain_retry call of this engine did not require DL_CHECK_RINGS";
  else if (B != e->ring_B) why = "B differs from the last dl_sample_chain_retry call's";
  if (why) { set_err("dl_last_ring_sizes: %s", why); return DL_ERR_INVALID; }
  CK(cudaMemcpyAsync(out, e->ring_masks.buf, (size_t)B * sizeof(uint64_t), cudaMemcpyDeviceToDevice,
                     reinterpret_cast<cudaStream_t>(stream)));
  return DL_OK;
}

float dl_last_retry_ms(dl_engine* e) { return e ? e->retry_ms : -1.f; }

int64_t dl_launch_count(const dl_engine* e) { return e ? e->launches : 0; }

int64_t dl_last_molecule_steps(dl_engine* e) { return e ? e->mol_steps : 0; }

float dl_last_elapsed_ms(dl_engine* e) {
  if (!e) return -1.f;
  float ms = -1.f;
  if (cudaEventElapsedTime(&ms, e->ev_t0, e->ev_t1) != cudaSuccess) { cudaGetLastError(); return -1.f; }
  return ms;
}

dl_status dl_cut_graph_stats(dl_engine* e, int64_t* out) {
  if (!e || !out) return DL_ERR_INVALID;
  Workspace& ws = e->ws;
  out[0] = out[1] = out[2] = out[3] = 0;
  if (ws.recs == nullptr) return DL_OK;
  if (cudaSetDevice(e->cfg.device) != cudaSuccess) return DL_ERR_CUDA;
  CK(cudaDeviceSynchronize());
  int n[2] = {0, 0};
  CK(cudaMemcpy(n, ws.n_recs, sizeof(n), cudaMemcpyDeviceToHost));
  std::vector<int> recs((size_t)n[0] * CUT_REC);
  CK(cudaMemcpy(recs.data(), ws.recs, recs.size() * sizeof(int), cudaMemcpyDeviceToHost));
  out[0] = n[0]; out[3] = n[1];
  long long n_heavy = 0, e_heavy = 0, max_heavy = 0, rows_light = 0;
  for (int k = 0; k < n[0]; ++k) {
    const int* r = recs.data() + (size_t)k * CUT_REC;
    const bool heavy = (r[1] >> 8) & 1;
    out[1] += heavy ? (r[2] + tc::TN - 1) / tc::TN : 1;
    out[2] += r[2];
    if (heavy) { ++n_heavy; e_heavy += r[2]; max_heavy = std::max<long long>(max_heavy, r[2]); }
    else rows_light += r[1] & 0xff;
  }
  if (getenv("DL_DEBUG_CUT"))
    fprintf(stderr, "[dl cut] records %d (heavy %lld, deg sum %lld, max %lld; light rows %lld) tiles %lld edges %lld | coord records %d\n",
            n[0], n_heavy, e_heavy, max_heavy, rows_light, (long long)out[1], (long long)out[2], n[1]);
  return DL_OK;
}

float dl_time_edge_kernel(dl_engine* e, int32_t reps) {
  if (!e || !e->finalized || e->last_B == 0 || reps < 1) { set_err("dl_time_edge_kernel: no previous forward"); return -1.f; }
  if (cudaSetDevice(e->cfg.device) != cudaSuccess) return -1.f;
  const Geom gm = make_geom(e, e->last_B, e->last_N);
  const GclW& w = e->gcl[0];
  // the forward's first GCL launch: block 0 reads the coordinates from ws.xa
  const EdgeArgs ea = edge_args(e, w, false, e->last_edge_mask, e->last_linker_mask, e->ws.xa, e->ws.xa4);
  cudaStream_t st = e->loop_stream;
  for (int i = 0; i < 2; ++i) if (launch_edge(e, gm, ea, false, w.W2_tc, st) != DL_OK) return -1.f;
  if (cudaEventRecord(e->ev_t0, st) != cudaSuccess) return -1.f;
  for (int i = 0; i < reps; ++i) if (launch_edge(e, gm, ea, false, w.W2_tc, st) != DL_OK) return -1.f;
  if (cudaEventRecord(e->ev_t1, st) != cudaSuccess) return -1.f;
  if (cudaStreamSynchronize(st) != cudaSuccess) { set_err("dl_time_edge_kernel: %s", cudaGetErrorString(cudaGetLastError())); return -1.f; }
  float ms = -1.f;
  if (cudaEventElapsedTime(&ms, e->ev_t0, e->ev_t1) != cudaSuccess) return -1.f;
  return ms / reps;
}

dl_status dl_selftest_tc(dl_engine* e, float* max_abs_err, float* max_rel_err) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  return tc::selftest(e->num_sms, max_abs_err, max_rel_err, false);
}

dl_status dl_selftest_tc_layout(dl_engine* e, int32_t b_mn_major, float* max_abs_err, float* max_rel_err) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  if (b_mn_major < 0 || b_mn_major > 1) { set_err("b_mn_major must be 0 (K-major B) or 1 (MN-major B)"); return DL_ERR_INVALID; }
  return tc::selftest(e->num_sms, max_abs_err, max_rel_err, b_mn_major != 0);
}

}  // extern "C"

#include "size_gnn.cuh"
