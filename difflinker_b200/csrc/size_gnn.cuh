// SizeGNN / SizeClassifier.forward (src/linker_size.py:45-91, src/linker_size_lightning.py:83-110): the linker-size
// classifier that runs once per batch right before the sampler (generate.py:88-99, SURVEY.md section 8(f) rank 3).
// Included at the end of dl_engine.cu: it is a second specialisation of the fp32 SIMT kernels of the denoiser
// (k_prep -> [k_edge_simt<GCL, ReLU> -> k_node<ReLU>] x n_layers -> k_sz_out):
//   x = positions * fragment_mask ; h = embedding_in(one_hot * fragment_mask)            (all rows, unmasked: + bias)
//   m_ij = relu(W2 relu(W1 [h_i, h_j, |x_i-x_j|^2] + b1) + b2) * (edge_mask_ij != 0 and |x_i-x_j|^2 < 6)
//   h = (h + W4 relu(W3 [h, sum_j m_ij] + b3) + b4) * fragment_mask          (normalization_factor = 1, 'sum')
//   out[b] = mean over the N padded rows of embedding_out(h)
// It is tiny next to the 500-step sampler (one pass over B*N^2 edges), so the fp32 SIMT kernels are the right tool.
// normalization='batch_norm' (eval mode) is an affine map per channel: the host folds it into W3/b3 and W4/b4.
// hidden_nf is 128 (the argparse default of train_size_gnn.py) or 256 (the reference README's recipe). The 256-wide model
// runs its own kernels (kernels_size_wide.cuh: k_szw_prep -> [k_szw_edge -> k_szw_node] x n_layers -> k_szw_out) with the
// same arithmetic, edge set and summation order; the 128-wide one runs the denoiser's SIMT kernels as before.
#include "kernels_size_wide.cuh"

struct dl_sizegnn {
  dl_sizegnn_config cfg{};
  int num_sms = 0;
  bool finalized = false;
  std::map<std::string, std::vector<float>> raw;
  float* wblob = nullptr;
  std::vector<GclW> layers;
  const float *We_t = nullptr, *be = nullptr, *Wo = nullptr, *bo = nullptr;
  Workspace ws;
  int64_t launches = 0;
};

namespace {

std::vector<ExpectedParam> sz_expected_params(const dl_sizegnn_config& c) {
  std::vector<ExpectedParam> v;
  const int H = c.hidden_nf;
  v.push_back({"embedding_in.weight", (int64_t)H * c.in_node_nf});
  v.push_back({"embedding_in.bias", H});
  char buf[64];
  for (int l = 0; l < c.n_layers; ++l) {
    snprintf(buf, sizeof(buf), "layer%d.", l);
    std::string p(buf);
    v.push_back({p + "edge_mlp.0.weight", (int64_t)H * (2 * H + 1)});
    v.push_back({p + "edge_mlp.0.bias", H});
    v.push_back({p + "edge_mlp.2.weight", (int64_t)H * H});
    v.push_back({p + "edge_mlp.2.bias", H});
    v.push_back({p + "node_mlp.0.weight", (int64_t)H * 2 * H});
    v.push_back({p + "node_mlp.0.bias", H});
    v.push_back({p + "node_mlp.2.weight", (int64_t)H * H});
    v.push_back({p + "node_mlp.2.bias", H});
  }
  v.push_back({"embedding_out.weight", (int64_t)c.out_node_nf * H});
  v.push_back({"embedding_out.bias", c.out_node_nf});
  return v;
}

dl_status sz_ensure_workspace(dl_sizegnn* e, int B, int N) {
  Workspace& ws = e->ws;
  if (ws.B == B && ws.N == N) return DL_OK;
  free_workspace(ws);
  const size_t n = (size_t)B * N;
  const int H = e->cfg.hidden_nf;
  dl_status s;
#define WSA(field, cnt) if ((s = dev_alloc(ws, &ws.field, (cnt))) != DL_OK) return s
  WSA(nm, n); WSA(x0, n * 3); WSA(xa, n * 3); WSA(h, n * H); WSA(ABg, n * 2 * H); WSA(ABgmax, n * 2); WSA(agg, n * H);
  WSA(cls, n); WSA(rowidx, n); WSA(colidx, n); WSA(xrowidx, n); WSA(nr, B); WSA(nc, B); WSA(nxr, B); WSA(n_items, 1);
  WSA(xmols, B); WSA(n_xmols, 1); WSA(items, n); WSA(xitems, n); WSA(n_xitems, 1);
#undef WSA
  ws.B = B; ws.N = N;
  return DL_OK;
}

// k-major fp32 copies of one 256-wide GCL (prefix p ends in '.'): the edge MLP's first Linear over [h_i, h_j, radial]
// split into W1a_t / W1b_t / b1 / wd, its second Linear W2_t / b2, and the node MLP W3_t ([h, agg] rows) / b3, W4_t / b4.
void sz_pack_wide_gcl(Packer& pk, GclW& w, const RawWeights& raw, const std::string& p) {
  constexpr int Hw = szw::W;
  const auto& W1 = raw.at(p + "edge_mlp.0.weight");
  pk.add(&w.W1a_t, transpose_block(W1, Hw, 2 * Hw + 1, 0, Hw));
  pk.add(&w.W1b_t, transpose_block(W1, Hw, 2 * Hw + 1, Hw, Hw));
  pk.add(&w.b1, raw.at(p + "edge_mlp.0.bias"));
  pk.add(&w.wd, column(W1, Hw, 2 * Hw + 1, 2 * Hw));
  pk.add(&w.W2_t, transpose_block(raw.at(p + "edge_mlp.2.weight"), Hw, Hw, 0, Hw));
  pk.add(&w.b2, raw.at(p + "edge_mlp.2.bias"));
  pk.add(&w.W3_t, transpose_block(raw.at(p + "node_mlp.0.weight"), Hw, 2 * Hw, 0, 2 * Hw));
  pk.add(&w.b3, raw.at(p + "node_mlp.0.bias"));
  pk.add(&w.W4_t, transpose_block(raw.at(p + "node_mlp.2.weight"), Hw, Hw, 0, Hw));
  pk.add(&w.b4, raw.at(p + "node_mlp.2.bias"));
}

// The 256-wide forward after the work plan: the same launch sequence as the 128-wide one, on the wide kernels.
dl_status sz_forward_wide(dl_sizegnn* e, const Geom& gm, const int8_t* fragment_mask, const float* xh, const int8_t* edge_mask,
                          float* out, cudaStream_t st) {
  Workspace& ws = e->ws;
  const int n = gm.B * gm.N, L = e->cfg.n_layers;
  // build_plan zeroes the first B*N*128 floats of agg; dead rows of the 256-wide aggregate must be exactly 0 as well
  CK(cudaMemsetAsync(ws.agg, 0, (size_t)n * szw::W * sizeof(float), st));
  const int node_blocks = (n + szw::TM - 1) / szw::TM;
  szw::PrepArgsW pa{};
  pa.xh = xh; pa.node_mask = fragment_mask; pa.We_t = e->We_t; pa.be = e->be; pa.proj = proj_of(e->layers[0]);
  pa.nm = ws.nm; pa.x0 = ws.x0; pa.h = ws.h; pa.AB = ws.ABg;
  szw::k_szw_prep<<<node_blocks, 256, 0, st>>>(gm, pa);
  LAUNCH_CHECK();
  const Plan plan = make_plan(ws);
  for (int l = 0; l < L; ++l) {
    const GclW& w = e->layers[l];
    EdgeArgs ea{};
    ea.AB = ws.ABg; ea.x0 = ws.x0; ea.edge_mask = edge_mask; ea.nm = ws.nm;
    ea.W2_t = w.W2_t; ea.b2 = w.b2; ea.wd = w.wd; ea.plan = plan; ea.agg = ws.agg;
    szw::k_szw_edge<<<2 * e->num_sms, 256, szw::EDGE_SMEM, st>>>(gm, ea);
    LAUNCH_CHECK();
    NodeArgs na{};
    na.h = ws.h; na.agg = ws.agg; na.nm = ws.nm; na.W3_t = w.W3_t; na.b3 = w.b3; na.W4_t = w.W4_t; na.b4 = w.b4;
    if (l + 1 < L) { na.proj1 = proj_of(e->layers[l + 1]); na.AB1 = ws.ABg; }
    szw::k_szw_node<<<node_blocks, 256, szw::NODE_SMEM, st>>>(n, na);
    LAUNCH_CHECK();
  }
  szw::k_szw_out<<<gm.B, 256, 0, st>>>(gm.N, e->cfg.out_node_nf, ws.h, e->Wo, e->bo, out);
  LAUNCH_CHECK();
  e->launches += 4 + 2 * L;
  return DL_OK;
}

}  // namespace

extern "C" {

dl_status dl_sizegnn_create(const dl_sizegnn_config* cfg, dl_sizegnn** out) {
  if (!cfg || !out) { set_err("null argument"); return DL_ERR_INVALID; }
  if (cfg->hidden_nf != H && cfg->hidden_nf != szw::W) {
    set_err("SizeGNN: hidden_nf must be %d or %d (got %d)", H, szw::W, cfg->hidden_nf);
    return DL_ERR_UNSUPPORTED;
  }
  if (cfg->in_node_nf < 1 || cfg->in_node_nf > MAX_DIN || cfg->n_layers < 1 || cfg->out_node_nf < 1 ||
      cfg->out_node_nf > SZ_MAX_OUT) {
    set_err("SizeGNN: unsupported shape (in_node_nf %d, n_layers %d, out_node_nf %d)", cfg->in_node_nf, cfg->n_layers,
            cfg->out_node_nf);
    return DL_ERR_UNSUPPORTED;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    set_err("no CUDA device: difflinker_b200 has no CPU fallback");
    return DL_ERR_CUDA;
  }
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop{};
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  dl_sizegnn* e = new dl_sizegnn();
  e->cfg = *cfg;
  e->num_sms = prop.multiProcessorCount;
  if (cfg->hidden_nf == szw::W) {
    CK(cudaFuncSetAttribute(szw::k_szw_node, cudaFuncAttributeMaxDynamicSharedMemorySize, szw::NODE_SMEM));
    CK(cudaFuncSetAttribute(szw::k_szw_edge, cudaFuncAttributeMaxDynamicSharedMemorySize, szw::EDGE_SMEM));
  } else {
    CK(cudaFuncSetAttribute(k_node<ACT_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, 3 * NODE_TM * LDX * sizeof(float)));
    CK(cudaFuncSetAttribute(k_edge_simt<false, ACT_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EDGE_SIMT_SMEM));
  }
  *out = e;
  return DL_OK;
}

dl_status dl_sizegnn_destroy(dl_sizegnn* e) {
  if (!e) return DL_OK;
  cudaSetDevice(e->cfg.device);
  cudaDeviceSynchronize();
  free_workspace(e->ws);
  if (e->wblob) cudaFree(e->wblob);
  delete e;
  return DL_OK;
}

dl_status dl_sizegnn_set_weight(dl_sizegnn* e, const char* name, const float* data, int64_t numel) {
  if (!e || !name || !data) { set_err("null argument"); return DL_ERR_INVALID; }
  for (auto& p : sz_expected_params(e->cfg)) {
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

dl_status dl_sizegnn_finalize_weights(dl_sizegnn* e) {
  if (!e) { set_err("null engine"); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  for (auto& p : sz_expected_params(e->cfg))
    if (!e->raw.count(p.name)) { set_err("missing weight %s", p.name.c_str()); return DL_ERR_WEIGHTS; }
  const int L = e->cfg.n_layers, F_in = e->cfg.in_node_nf;
  const RawWeights& raw = e->raw;
  Packer pk;
  e->layers.assign(L, GclW{});
  const bool wide = e->cfg.hidden_nf == szw::W;
  pk.add(&e->We_t, transpose_block(raw.at("embedding_in.weight"), e->cfg.hidden_nf, F_in, 0, F_in));
  pk.add(&e->be, raw.at("embedding_in.bias"));
  pk.add(&e->Wo, raw.at("embedding_out.weight"));
  pk.add(&e->bo, raw.at("embedding_out.bias"));
  char buf[64];
  for (int l = 0; l < L; ++l) {
    snprintf(buf, sizeof(buf), "layer%d.", l);
    GclW& w = e->layers[l];
    if (wide) { sz_pack_wide_gcl(pk, w, raw, buf); continue; }
    pack_gcl(pk, w, raw, buf, 2 * H + 1);
    pk.add(&w.w0, std::vector<float>(H, 0.f));   // no input-distance column
  }
  const dl_status s = upload_blob(pk.blob, &e->wblob);
  if (s != DL_OK) return s;
  pk.point(e->wblob, nullptr);
  e->finalized = true;
  return DL_OK;
}

dl_status dl_sizegnn_forward(dl_sizegnn* e, int32_t B, int32_t N, const float* xh, const int8_t* fragment_mask,
                             const int8_t* edge_mask, float* out, void* stream) {
  if (!e || !e->finalized) { set_err("SizeGNN engine not finalized"); return DL_ERR_INVALID; }
  if (B <= 0 || N <= 0 || !xh || !fragment_mask || !out) { set_err("dl_sizegnn_forward: bad argument"); return DL_ERR_INVALID; }
  CK(cudaSetDevice(e->cfg.device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  dl_status s = sz_ensure_workspace(e, B, N);
  if (s != DL_OK) return s;
  Workspace& ws = e->ws;
  const int n = B * N, L = e->cfg.n_layers;
  Geom gm{};
  gm.B = B; gm.N = N; gm.F = e->cfg.in_node_nf; gm.C = 0; gm.D = e->cfg.in_node_nf;
  gm.graph_type = 4; gm.norm_constant = 0.f; gm.normalization_factor = 1.f;

  if ((s = build_plan(ws, B, N, gm.graph_type, fragment_mask, nullptr, edge_mask, ET, MAXR, st)) != DL_OK) return s;
  if (e->cfg.hidden_nf == szw::W) return sz_forward_wide(e, gm, fragment_mask, xh, edge_mask, out, st);

  const int node_blocks = (n + NODE_TM - 1) / NODE_TM;
  PrepArgs pa{};
  pa.xh = xh; pa.node_mask = fragment_mask; pa.linker_mask = nullptr; pa.t = nullptr; pa.t_numel = 0; pa.context = nullptr;
  pa.We_t = e->We_t; pa.be = e->be;
  pa.proj = proj_of(e->layers[0]);
  pa.nm = ws.nm; pa.x0 = ws.x0; pa.x = ws.xa; pa.x04 = nullptr; pa.x4 = nullptr; pa.cls = ws.cls; pa.h = ws.h;
  pa.AB = ws.ABg; pa.ABmax = ws.ABgmax;
  k_prep<<<node_blocks, 256, 0, st>>>(gm, pa);
  LAUNCH_CHECK();

  const Plan plan = make_plan(ws);
  const size_t node_smem = 3 * NODE_TM * LDX * sizeof(float);
  for (int l = 0; l < L; ++l) {
    const GclW& w = e->layers[l];
    EdgeArgs ea{};
    ea.AB = ws.ABg; ea.ABmax = ws.ABgmax; ea.x = ws.xa; ea.x0 = ws.x0; ea.edge_mask = edge_mask; ea.cls = ws.cls; ea.nm = ws.nm;
    ea.W2_t = w.W2_t; ea.b2 = w.b2; ea.wd = w.wd; ea.w0 = w.w0; ea.plan = plan; ea.agg = ws.agg;
    k_edge_simt<false, ACT_RELU><<<e->num_sms, 256, EDGE_SIMT_SMEM, st>>>(gm, ea);
    LAUNCH_CHECK();
    NodeArgs na{};
    na.h = ws.h; na.agg = ws.agg; na.nm = ws.nm; na.W3_t = w.W3_t; na.b3 = w.b3; na.W4_t = w.W4_t; na.b4 = w.b4;
    if (l + 1 < L) {
      na.proj1 = proj_of(e->layers[l + 1]); na.AB1 = ws.ABg; na.ABmax1 = ws.ABgmax;
    }
    k_node<ACT_RELU><<<node_blocks, 256, node_smem, st>>>(n, na);
    LAUNCH_CHECK();
  }
  k_sz_out<<<B, 256, 0, st>>>(N, e->cfg.out_node_nf, ws.h, e->Wo, e->bo, out);
  LAUNCH_CHECK();
  e->launches += 4 + 2 * L;
  return DL_OK;
}

}  // extern "C"
