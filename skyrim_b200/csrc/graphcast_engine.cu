// GraphCast 6-h step operator on sm_90a (SURVEY.md §8(a) A9 / §8(f) N1): replaces what Skyrim's GraphCast model
// (skyrim/core/models/graphcast.py, `self.stepper.step(state)`) runs inside earth2mip's JAX wrapper.
//
// State tensor of one member: (2 x 83, nlat, nlon) fp32 = the two time slices (t-6h, t) of the reference's 83-channel
// field (graphcast.py:17-41; 82 prognostic channels + the toa-radiation forcing the reference labels "tp06").
// One step = encoder (grid -> mesh), 16 message-passing layers on the multimesh, decoder (mesh -> grid), residual update.
//
// H100 mapping.  Every MLP is two persistent TMA-fed wgmma GEMMs: hidden = swish(A W1^T + ...) (k_gemm2) written as the
// fp16 operand image of the second GEMM (k_gemm2_pair: column-split CTA pairs of a cluster, LayerNorm statistics over
// DSMEM), whose epilogue does bias + LayerNorm (+ residual, read from the
// stream's own fp16 image for grid nodes and mesh edges) and writes the operand image of whatever consumes it next.  The concatenations of the published formulation never exist:
//   * [edge, sender, receiver] W1^T = edge W1e^T + (v W1s^T)[sender] + (v W1r^T)[receiver]: the per-NODE products are
//     small GEMMs into fp16 tables, gathered by edge index inside the hidden GEMM's epilogue (row-owner lanes);
//   * [node, sum of incoming edges] is a K-concatenation of two operand images (AOperand), the sum produced by a
//     deterministic CSR reduction over the edge-update image (mesh, grid2mesh) or, for mesh2grid where every grid point has
//     exactly three incoming edges stored k-major, by a K-concatenation of the three edge-update images with W1a repeated;
//   * embeddings of mesh nodes and of the three edge sets do not depend on the input: computed once at load.
// Members of a batch are processed one after the other (weights stay in L2 between members; config 4 is single member).
#include <cstdio>
#include <cstring>
#include <vector>

#include "engine.h"
#include "graphcast_ops.cuh"

namespace sky {

static inline long long pad128(long long r) { return (r + 127) / 128 * 128; }
static inline size_t img_bytes(long long rows, int nkb) { return (size_t)(pad128(rows) / 128) * nkb * G2_A_BYTES; }

struct WImg { uint8_t* img = nullptr; int N = 0, Kp = 0, BN = 0; };
struct Mlp {
  WImg w1, w2;
  WImg w2s;   // second layer of the LayerNorm MLPs, packed in 256-row halves for the column-split pair kernel (k_gemm2_pair)
  const float *b1 = nullptr, *b2 = nullptr, *g = nullptr, *be = nullptr;
};

struct GraphCastEngine : Engine {
  sky_graphcast_config_t cfg;
  long long Ng, Ngp, Nm, Em, Eg, E3;   // grid points (padded to row tiles), mesh nodes, mesh / grid2mesh / mesh2grid rows
  int nfeat;
  std::vector<void*> owned;
  // parameters
  Mlp grid_embed, g2m_edge, g2m_mesh, g2m_grid, m2g_edge, m2g_grid, out_mlp;
  std::vector<Mlp> proc_edge, proc_node;
  WImg g2m_ws, m2g_ws, m2g_wr;          // per-node first-layer tables: (N = 512, K = 512)
  std::vector<WImg> proc_wsr;           // (N = 1024: [W1s; W1r], K = 512)
  const float *mean = nullptr, *stdv = nullptr, *dstd = nullptr, *statics = nullptr, *zero_bias = nullptr;
  // graph
  int *mesh_s = nullptr, *mesh_r = nullptr, *g2m_s = nullptr, *g2m_r = nullptr, *m2g_s = nullptr, *m2g_r = nullptr;
  struct SegPlan {   // chunked CSR reduction (k_gc_segsum): chunk table, cut nodes, fp32 partial rows
    GcSegChunk* chunks = nullptr; int n_chunks = 0;
    GcSegMulti* multi = nullptr; int n_multi = 0;
    float* partial = nullptr;
  } mesh_seg, g2m_seg;
  // input-independent embeddings
  uint8_t *e_g2m_img = nullptr, *e_m2g_img = nullptr, *e_mesh_img = nullptr, *vm0_img = nullptr;
  float* vm0_f32 = nullptr;
  __half* g2m_tr = nullptr;             // (Nm, 512): embedded mesh nodes x W1r(g2m_edge)^T
  cudaStream_t prep_stream = nullptr;   // stream of the running prepare() (dalloc's zero fills)
  // clock
  double* clock_dev = nullptr;
  GcClock* clk_dev = nullptr;

  GraphCastEngine(const sky_graphcast_config_t& c, int dev) : cfg(c) {
    device = dev;
    Ng = (long long)c.nlat * c.nlon;
    Ngp = pad128(Ng);
    Nm = c.n_mesh; Em = c.n_mesh_edges; Eg = c.n_g2m_edges; E3 = 3 * Ngp;
    nfeat = 2 * c.n_prog + 3 + 12 + c.n_static + 3;
  }
  ~GraphCastEngine() override { for (void* p : owned) cudaFree(p); }

  template <class T>
  T* dalloc(size_t n, bool zero = false) {
    void* p = nullptr;
    if (cudaMalloc(&p, n * sizeof(T) + 16) != cudaSuccess) { set_error("cudaMalloc(%zu) failed", n * sizeof(T)); return nullptr; }
    // zero-fill on the stream the packing kernels run on (a legacy-stream cudaMemset is not ordered against a non-blocking stream)
    if (zero) cudaMemsetAsync(p, 0, n * sizeof(T) + 16, prep_stream);
    owned.push_back(p);
    return reinterpret_cast<T*>(p);
  }
  void dfree(void* p) {
    for (size_t i = 0; i < owned.size(); ++i) if (owned[i] == p) { owned.erase(owned.begin() + i); break; }
    cudaFree(p);
  }

  // ---- weight packing ------------------------------------------------------------------------------------------
  int walloc(WImg& w, int N, int K, int BN) {
    w.N = (N + BN - 1) / BN * BN; w.Kp = (K + 63) / 64 * 64; w.BN = BN;
    w.img = dalloc<uint8_t>((size_t)w.N * w.Kp * 2, true);
    return w.img ? 0 : SKY_ERR_NOMEM;
  }
  // columns [c0, c0 + K) of the (N, ldw) parameter `name` -> columns [k_off, ..) of rows [n_off, ..) of w
  int wfill(WImg& w, const char* name, int N, int ldw, int c0, int K, int k_off, int n_off, cudaStream_t st) {
    const float* src = param(name, (uint64_t)N * ldw);
    if (!src) return SKY_ERR_ARG;
    const long long chunks = (long long)N * ((K + 7) / 8);
    k_gc_pack_w<<<(unsigned)((chunks + 255) / 256), 256, 0, st>>>(src, ldw, c0, N, K, k_off, w.Kp, w.BN, n_off, w.img);
    count_launch();
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }
  int load_mlp(Mlp& m, const char* name, int fan_in, int k_in /*columns of w1 kept in the A-operand GEMM*/, int fan_out, bool ln,
               cudaStream_t st, int w2_bn = 256) {
    char nm[96];
    auto N = [&](const char* s) { snprintf(nm, sizeof nm, "%s.%s", name, s); return nm; };
    int rc;
    if (k_in > 0) {
      if ((rc = walloc(m.w1, GC_L, k_in, 256))) return rc;
      if ((rc = wfill(m.w1, N("w1"), GC_L, fan_in, 0, k_in, 0, 0, st))) return rc;
    }
    if (ln && fan_out == GC_L) {   // LayerNorm over 512 columns: column-split pair kernel, 256-row halves
      if ((rc = walloc(m.w2s, GC_L, GC_L, 256))) return rc;
      if ((rc = wfill(m.w2s, N("w2"), GC_L, GC_L, 0, GC_L, 0, 0, st))) return rc;
    } else {
      if ((rc = walloc(m.w2, fan_out, GC_L, w2_bn))) return rc;
      if ((rc = wfill(m.w2, N("w2"), fan_out, GC_L, 0, GC_L, 0, 0, st))) return rc;
    }
    if (!(m.b1 = keep(N("b1"), GC_L, st))) return SKY_ERR_ARG;
    {   // b2 / gamma / beta padded to the n-tile width (the kernel stages BLOCK_N entries)
      const float* b2 = param(N("b2"), (uint64_t)fan_out);
      if (!b2) return SKY_ERR_ARG;
      float* p = dalloc<float>((size_t)(m.w2.img ? m.w2.N : m.w2s.N), true);
      if (!p) return SKY_ERR_NOMEM;
      SKY_CUDA_OK(cudaMemcpyAsync(p, b2, (size_t)fan_out * 4, cudaMemcpyDeviceToDevice, st));
      m.b2 = p;
    }
    if (ln) {
      if (!(m.g = keep(N("ln.g"), (uint64_t)fan_out, st))) return SKY_ERR_ARG;
      if (!(m.be = keep(N("ln.b"), (uint64_t)fan_out, st))) return SKY_ERR_ARG;
    }
    return 0;
  }
  // receiver-sorted edge list -> chunk table (segments cut at GC_SEG_CHUNK edges).  Built on the host from the CSR pointer.
  int load_segplan(SegPlan& sp, const char* ptr_name, long long n_nodes, cudaStream_t st) {
    const float* src = param(ptr_name, (uint64_t)n_nodes + 1);
    if (!src) return SKY_ERR_ARG;
    std::vector<float> hp((size_t)n_nodes + 1);
    SKY_CUDA_OK(cudaMemcpyAsync(hp.data(), src, hp.size() * 4, cudaMemcpyDeviceToHost, st));
    SKY_CUDA_OK(cudaStreamSynchronize(st));
    std::vector<GcSegChunk> ck;
    std::vector<GcSegMulti> mu;
    int parts = 0;
    for (long long n = 0; n < n_nodes; ++n) {
      const int e0 = (int)hp[n], e1 = (int)hp[n + 1];
      const int nc = e1 - e0 <= GC_SEG_CHUNK ? 1 : (e1 - e0 + GC_SEG_CHUNK - 1) / GC_SEG_CHUNK;
      if (nc == 1) { ck.push_back(GcSegChunk{(int)n, e0, e1, -1}); continue; }
      mu.push_back(GcSegMulti{(int)n, parts, parts + nc});
      for (int c = 0; c < nc; ++c) {
        const int a = e0 + c * GC_SEG_CHUNK;
        ck.push_back(GcSegChunk{(int)n, a, a + GC_SEG_CHUNK < e1 ? a + GC_SEG_CHUNK : e1, parts++});
      }
    }
    sp.n_chunks = (int)ck.size(); sp.n_multi = (int)mu.size();
    sp.chunks = dalloc<GcSegChunk>(ck.size());
    if (!sp.chunks) return SKY_ERR_NOMEM;
    SKY_CUDA_OK(cudaMemcpyAsync(sp.chunks, ck.data(), ck.size() * sizeof(GcSegChunk), cudaMemcpyHostToDevice, st));
    if (sp.n_multi) {
      sp.multi = dalloc<GcSegMulti>(mu.size());
      sp.partial = dalloc<float>((size_t)parts * GC_L);
      if (!sp.multi || !sp.partial) return SKY_ERR_NOMEM;
      SKY_CUDA_OK(cudaMemcpyAsync(sp.multi, mu.data(), mu.size() * sizeof(GcSegMulti), cudaMemcpyHostToDevice, st));
    }
    SKY_CUDA_OK(cudaStreamSynchronize(st));   // the host vectors die here
    return 0;
  }
  int load_index(int*& dst, const char* name, long long n, cudaStream_t st) {
    const float* src = param(name, (uint64_t)n);
    if (!src) return SKY_ERR_ARG;
    dst = dalloc<int>((size_t)n);
    if (!dst) return SKY_ERR_NOMEM;
    k_gc_f2i<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, dst, n);
    count_launch();
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }

  // ---- GEMM wrappers --------------------------------------------------------------------------------------------
  template <int kG>
  int hidden(int tag, const AOperand& A, int Kp, const WImg& w, const float* b1, long long M, uint8_t* out, const __half* ta, int lda,
             const int* ia, const __half* tb, int ldb, const int* ib, cudaStream_t st) {
    if (w.BN != 256 || w.Kp != Kp) { set_error("internal: hidden GEMM weight shape"); return SKY_ERR_STATE; }
    EpiGcSiluImg<kG> epi{};
    epi.out = out; epi.bias = b1; epi.ta = ta; epi.lda = lda; epi.ia = ia; epi.tb = tb; epi.ldb = ldb; epi.ib = ib;
    prof_begin(tag, st);
    count_launch();
    const int rc = launch_gemm2<256>(SchedW<>{A, w.img, Kp / 64}, epi, M, GC_L, 1, num_sms, st);
    prof_end(tag, st);
    // fp16-range guard (engine.h; a no-op unless enabled): class 5 hidden images, 0 latent / update images, 6 per-node tables
    return rc ? rc : range_scan(5, out, (size_t)(M / 128) * GC_NKB * G2_A_BYTES, st);
  }
  template <int kRes>
  int ln_launch(const uint8_t* hid, const Mlp& m, long long M, const float* xin, float* xout, uint8_t* img, uint8_t* yimg,
                const uint8_t* xin_img, cudaStream_t st) {
    EpiGcLn<kRes> epi{xin, xout, img, yimg, m.b2, m.g, m.be, cfg.ln_eps};
    epi.xin_img = xin_img;
    return launch_gemm2<256, true>(SchedW<>{AOperand(hid, GC_NKB), m.w2s.img, GC_NKB}, epi, M, GC_L, 1, num_sms, st);
  }
  // xin (fp32 rows) or xin_img (fp16 image) is the residual source; at most one of them
  int ln_gemm(int tag, const uint8_t* hid, const Mlp& m, long long M, const float* xin, float* xout, uint8_t* img, uint8_t* yimg,
              cudaStream_t st, const uint8_t* xin_img = nullptr) {
    prof_begin(tag, st);
    count_launch();
    int rc;
    if (xin) rc = ln_launch<1>(hid, m, M, xin, xout, img, yimg, nullptr, st);
    else if (xin_img) rc = ln_launch<2>(hid, m, M, nullptr, xout, img, yimg, xin_img, st);
    else rc = ln_launch<0>(hid, m, M, nullptr, xout, img, yimg, nullptr, st);
    prof_end(tag, st);
    if (rc) return rc;
    if (img) if (int r2 = range_scan(0, img, (size_t)(M / 128) * GC_NKB * G2_A_BYTES, st)) return r2;
    return yimg ? range_scan(0, yimg, (size_t)(M / 128) * GC_NKB * G2_A_BYTES, st) : 0;
  }
  // per-node table: T (M, N) fp16 row-major = A W^T
  int table(int tag, const uint8_t* aimg, const WImg& w, long long M, __half* out, cudaStream_t st) {
    Epi2F16<false, false> epi{};
    epi.out = out; epi.ldo = w.N; epi.nkb = 0; epi.bias = zero_bias;
    prof_begin(tag, st);
    count_launch();
    const int rc = launch_gemm2<256>(SchedW<>{AOperand(aimg, GC_NKB), w.img, GC_NKB}, epi, M, w.N, 1, num_sms, st);
    prof_end(tag, st);
    return rc ? rc : range_scan(6, out, (size_t)M * w.N * 2, st);
  }
  int segsum(int tag, const uint8_t* yimg, const SegPlan& sp, uint8_t* out, cudaStream_t st) {
    prof_begin(tag, st);
    count_launch();
    k_gc_segsum<<<(unsigned)(((long long)sp.n_chunks * 32 + 255) / 256), 256, 0, st>>>(yimg, sp.chunks, sp.n_chunks, out, sp.partial);
    prof_end(tag, st);
    if (sp.n_multi) {
      prof_begin(tag, st);
      count_launch();
      k_gc_segsum_fin<<<(unsigned)(((long long)sp.n_multi * 32 + 255) / 256), 256, 0, st>>>(sp.partial, sp.multi, sp.n_multi, out);
      prof_end(tag, st);
    }
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }

  // ---- load: parameters, graph tables, input-independent embeddings ------------------------------------------
  // MLP(features F <= 64) of `rows` static rows -> image (and fp32 rows) of the embedding
  int static_embed(const char* name, const float* feat_dev, long long rows, int F, uint8_t* out_img, float* out_f32, cudaStream_t st) {
    Mlp m;
    int rc = load_mlp(m, name, F, F, GC_L, true, st);
    if (rc) return rc;
    uint8_t* fimg = dalloc<uint8_t>(img_bytes(rows, 1), true);
    uint8_t* hid = dalloc<uint8_t>(img_bytes(rows, GC_NKB));
    if (!fimg || !hid) return SKY_ERR_NOMEM;
    k_gc_pack_rows<<<(unsigned)((rows * 8 + 255) / 256), 256, 0, st>>>(feat_dev, rows, F, fimg);
    count_launch();
    if ((rc = hidden<0>(KT_GC_MISC, AOperand(fimg, 1), 64, m.w1, m.b1, rows, hid, nullptr, 0, nullptr, nullptr, 0, nullptr, st))) return rc;
    if ((rc = ln_gemm(KT_GC_MISC, hid, m, rows, nullptr, out_f32, out_img, nullptr, st))) return rc;
    SKY_CUDA_OK(cudaStreamSynchronize(st));
    dfree(fimg); dfree(hid); dfree(m.w1.img); dfree(m.w2.img); dfree(m.w2s.img); dfree(const_cast<float*>(m.b2));
    return 0;
  }

  int prepare(cudaStream_t st) override {
    prep_stream = st;
    if (cfg.latent != GC_L) { set_error("GraphCast engine is built for latent %d", GC_L); return SKY_ERR_ARG; }
    if (nfeat > GC_FEAT_KP || cfg.n_state != cfg.n_prog + 1) { set_error("unsupported GraphCast channel layout"); return SKY_ERR_ARG; }
    const int L = GC_L;
    int rc;
#define P(dst, name, cnt) if (!((dst) = keep(name, (uint64_t)(cnt), st))) return SKY_ERR_ARG;
    P(mean, "norm.mean", cfg.n_state); P(stdv, "norm.std", cfg.n_state); P(dstd, "norm.diff_std", cfg.n_state);
    P(statics, "static.fields", (long long)cfg.n_static * Ng);
#undef P
    { float* z = dalloc<float>(1024, true); if (!z) return SKY_ERR_NOMEM; zero_bias = z; }
    clock_dev = dalloc<double>(2, true);
    clk_dev = dalloc<GcClock>(1, true);
    if (!clock_dev || !clk_dev) return SKY_ERR_NOMEM;
    // ---- graph tables
    if ((rc = load_index(mesh_s, "graph.mesh.senders", Em, st))) return rc;
    if ((rc = load_index(mesh_r, "graph.mesh.receivers", Em, st))) return rc;
    if ((rc = load_segplan(mesh_seg, "graph.mesh.ptr", Nm, st))) return rc;
    if ((rc = load_index(g2m_s, "graph.g2m.senders", Eg, st))) return rc;
    if ((rc = load_index(g2m_r, "graph.g2m.receivers", Eg, st))) return rc;
    if ((rc = load_segplan(g2m_seg, "graph.g2m.ptr", Nm, st))) return rc;
    {
      const float* s = param("graph.m2g.senders", (uint64_t)3 * Ng);
      if (!s) return SKY_ERR_ARG;
      m2g_s = dalloc<int>((size_t)E3); m2g_r = dalloc<int>((size_t)E3);
      if (!m2g_s || !m2g_r) return SKY_ERR_NOMEM;
      k_gc_m2g_index<<<(unsigned)((E3 + 255) / 256), 256, 0, st>>>(s, m2g_s, m2g_r, Ng, Ngp);
      count_launch();
    }
    // ---- MLPs of the step
    if ((rc = load_mlp(grid_embed, "enc.grid_embed", nfeat, nfeat, L, true, st))) return rc;
    if ((rc = load_mlp(g2m_edge, "enc.g2m_edge", 3 * L, L, L, true, st))) return rc;
    if ((rc = load_mlp(g2m_mesh, "enc.g2m_mesh", 2 * L, 2 * L, L, true, st))) return rc;
    if ((rc = load_mlp(g2m_grid, "enc.g2m_grid", L, L, L, true, st))) return rc;
    if ((rc = walloc(g2m_ws, L, L, 256)) || (rc = wfill(g2m_ws, "enc.g2m_edge.w1", L, 3 * L, L, L, 0, 0, st))) return rc;
    proc_edge.resize(cfg.layers); proc_node.resize(cfg.layers); proc_wsr.resize(cfg.layers);
    for (int i = 0; i < cfg.layers; ++i) {
      char nm[64], nw[80];
      snprintf(nm, sizeof nm, "proc%d.edge", i);
      if ((rc = load_mlp(proc_edge[i], nm, 3 * L, L, L, true, st))) return rc;
      snprintf(nw, sizeof nw, "proc%d.edge.w1", i);
      if ((rc = walloc(proc_wsr[i], 2 * L, L, 256))) return rc;
      if ((rc = wfill(proc_wsr[i], nw, L, 3 * L, L, L, 0, 0, st))) return rc;        // rows 0..511:   W1s
      if ((rc = wfill(proc_wsr[i], nw, L, 3 * L, 2 * L, L, 0, L, st))) return rc;    // rows 512..1023: W1r
      snprintf(nm, sizeof nm, "proc%d.node", i);
      if ((rc = load_mlp(proc_node[i], nm, 2 * L, 2 * L, L, true, st))) return rc;
    }
    if ((rc = load_mlp(m2g_edge, "dec.m2g_edge", 3 * L, L, L, true, st))) return rc;
    if ((rc = walloc(m2g_ws, L, L, 256)) || (rc = wfill(m2g_ws, "dec.m2g_edge.w1", L, 3 * L, L, L, 0, 0, st))) return rc;
    if ((rc = walloc(m2g_wr, L, L, 256)) || (rc = wfill(m2g_wr, "dec.m2g_edge.w1", L, 3 * L, 2 * L, L, 0, 0, st))) return rc;
    // grid update of the decoder: [v | e0 | e1 | e2] x [W1v | W1a | W1a | W1a]^T
    if ((rc = load_mlp(m2g_grid, "dec.m2g_grid", 2 * L, 0, L, true, st))) return rc;
    if ((rc = walloc(m2g_grid.w1, L, 4 * L, 256))) return rc;
    if ((rc = wfill(m2g_grid.w1, "dec.m2g_grid.w1", L, 2 * L, 0, L, 0, 0, st))) return rc;
    for (int k = 0; k < 3; ++k)
      if ((rc = wfill(m2g_grid.w1, "dec.m2g_grid.w1", L, 2 * L, L, L, (1 + k) * L, 0, st))) return rc;
    if ((rc = load_mlp(out_mlp, "dec.out", L, L, cfg.n_state, false, st, 128))) return rc;
    // ---- input-independent embeddings
    e_g2m_img = dalloc<uint8_t>(img_bytes(Eg, GC_NKB), true);
    e_m2g_img = dalloc<uint8_t>(img_bytes(E3, GC_NKB), true);
    e_mesh_img = dalloc<uint8_t>(img_bytes(Em, GC_NKB), true);
    vm0_img = dalloc<uint8_t>(img_bytes(Nm, GC_NKB), true);
    vm0_f32 = dalloc<float>((size_t)pad128(Nm) * L, true);
    g2m_tr = dalloc<__half>((size_t)pad128(Nm) * L, true);
    if (!e_g2m_img || !e_m2g_img || !e_mesh_img || !vm0_img || !vm0_f32 || !g2m_tr) return SKY_ERR_NOMEM;
    const float* f;
    if (!(f = param("graph.mesh.node_feat", (uint64_t)Nm * 3))) return SKY_ERR_ARG;
    if ((rc = static_embed("enc.mesh_embed", f, Nm, 3, vm0_img, vm0_f32, st))) return rc;
    if (!(f = param("graph.g2m.edge_feat", (uint64_t)Eg * 4))) return SKY_ERR_ARG;
    if ((rc = static_embed("enc.g2m_edge_embed", f, Eg, 4, e_g2m_img, nullptr, st))) return rc;
    if (!(f = param("graph.mesh.edge_feat", (uint64_t)Em * 4))) return SKY_ERR_ARG;
    if ((rc = static_embed("proc.edge_embed", f, Em, 4, e_mesh_img, nullptr, st))) return rc;
    {
      if (!(f = param("graph.m2g.edge_feat", (uint64_t)3 * Ng * 4))) return SKY_ERR_ARG;
      float* fp = dalloc<float>((size_t)E3 * 4);
      if (!fp) return SKY_ERR_NOMEM;
      k_gc_m2g_feat<<<(unsigned)((E3 + 255) / 256), 256, 0, st>>>(f, fp, Ng, Ngp);
      count_launch();
      if ((rc = static_embed("dec.m2g_edge_embed", fp, E3, 4, e_m2g_img, nullptr, st))) return rc;
      dfree(fp);
    }
    {   // receiver table of the grid2mesh edge update: embedded mesh nodes x W1r^T (input independent)
      WImg wr;
      if ((rc = walloc(wr, L, L, 256)) || (rc = wfill(wr, "enc.g2m_edge.w1", L, 3 * L, 2 * L, L, 0, 0, st))) return rc;
      if ((rc = table(KT_GC_MISC, vm0_img, wr, Nm, g2m_tr, st))) return rc;
      SKY_CUDA_OK(cudaStreamSynchronize(st));
      dfree(wr.img);
    }
    SKY_CUDA_OK(cudaGetLastError());
    SKY_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  }

  // ---- workspace --------------------------------------------------------------------------------------------------
  struct Ws {
    uint8_t *feat, *hid, *vg_img, *yimg, *vm_img, *em_img, *ym_img, *agg_img, *hid_m;
    float* vm;
    __half *tg, *tm;
    size_t total;
  };
  Ws carve(void* base) const {
    Ws w;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 1023) / 1024 * 1024; return (char*)base + o; };
    const long long Emax = E3 > pad128(Eg) ? E3 : pad128(Eg);
    w.feat = (uint8_t*)take(img_bytes(Ng, GC_FEAT_KP / 64));
    w.hid = (uint8_t*)take(img_bytes(Emax, GC_NKB));          // hidden activations of the grid-sized / edge-sized MLPs
    w.vg_img = (uint8_t*)take(img_bytes(Ng, GC_NKB));
    w.tg = (__half*)take((size_t)Ngp * GC_L * 2);              // grid-node table (g2m sender / m2g receiver)
    w.yimg = (uint8_t*)take(img_bytes(Emax, GC_NKB));          // edge updates of the grid2mesh / mesh2grid step
    w.vm = (float*)take((size_t)pad128(Nm) * GC_L * 4);
    w.vm_img = (uint8_t*)take(img_bytes(Nm, GC_NKB));
    w.tm = (__half*)take((size_t)pad128(Nm) * 2 * GC_L * 2);   // mesh-node table [W1s | W1r]
    w.em_img = (uint8_t*)take(img_bytes(Em, GC_NKB));
    w.ym_img = (uint8_t*)take(img_bytes(Em, GC_NKB));
    w.agg_img = (uint8_t*)take(img_bytes(Nm, GC_NKB));
    w.hid_m = (uint8_t*)take(img_bytes(Em, GC_NKB));
    w.total = off;
    return w;
  }
  size_t workspace_bytes(int) const override { return carve(nullptr).total; }   // members run one after the other

  int set_clock(double unix_seconds, cudaStream_t st) override {
    if (!clock_dev) { set_error("set_clock before load_weights"); return SKY_ERR_STATE; }
    clock_host = unix_seconds;
    SKY_CUDA_OK(cudaMemcpyAsync(clock_dev, &clock_host, sizeof(double), cudaMemcpyHostToDevice, st));
    SKY_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  }
  double clock_host = 0.0;

  // ---- the step -----------------------------------------------------------------------------------------------------
  int step(const float* x_in, float* x_out, int batch, void* ws_base, size_t ws_bytes, cudaStream_t st) override {
    if (!loaded) { set_error("weights not loaded"); return SKY_ERR_STATE; }
    const Ws w = carve(ws_base);
    if (ws_bytes < w.total) { set_error("workspace too small: %zu < %zu", ws_bytes, w.total); return SKY_ERR_ARG; }
    const int L = GC_L;
    const long long plane = Ng;
    int rc;
    prof_begin(KT_GC_FEAT, st);
    count_launch();
    k_gc_clock<<<1, 32, 0, st>>>(clock_dev, clk_dev, 3600.0 * cfg.dt_hours, 1);
    prof_end(KT_GC_FEAT, st);
    for (int b = 0; b < batch; ++b) {
      const float* xi = x_in + (size_t)b * 2 * cfg.n_state * plane;
      float* xo = x_out + (size_t)b * 2 * cfg.n_state * plane;
      // ---------------- encoder
      prof_begin(KT_GC_FEAT, st);
      count_launch();
      k_gc_features<<<(unsigned)(Ngp / 128), 128, 0, st>>>(xi, xo, w.feat, mean, stdv, statics, clk_dev, cfg.nlat, cfg.nlon,
                                                            cfg.n_state, cfg.n_prog, cfg.n_static);
      prof_end(KT_GC_FEAT, st);
      SKY_CUDA_OK(cudaGetLastError());
      if ((rc = hidden<0>(KT_GC_HIDDEN, AOperand(w.feat, GC_FEAT_KP / 64), GC_FEAT_KP, grid_embed.w1, grid_embed.b1, Ng, w.hid, nullptr, 0, nullptr,
                          nullptr, 0, nullptr, st))) return rc;
      if ((rc = ln_gemm(KT_GC_LN, w.hid, grid_embed, Ng, nullptr, nullptr, w.vg_img, nullptr, st))) return rc;
      if (stop_after == 0) continue;
      if ((rc = table(KT_GC_TABLE, w.vg_img, g2m_ws, Ng, w.tg, st))) return rc;
      if ((rc = hidden<2>(KT_GC_HIDDEN, AOperand(e_g2m_img, GC_NKB), L, g2m_edge.w1, g2m_edge.b1, Eg, w.hid, w.tg, L, g2m_s, g2m_tr, L, g2m_r, st))) return rc;
      if ((rc = ln_gemm(KT_GC_LN, w.hid, g2m_edge, Eg, nullptr, nullptr, nullptr, w.yimg, st))) return rc;
      if ((rc = segsum(KT_GC_AGG, w.yimg, g2m_seg, w.agg_img, st))) return rc;
      if ((rc = hidden<0>(KT_GC_HIDDEN, AOperand(vm0_img, GC_NKB).add(w.agg_img, GC_NKB), 2 * L, g2m_mesh.w1, g2m_mesh.b1, Nm, w.hid_m, nullptr, 0, nullptr, nullptr, 0, nullptr, st))) return rc;
      if ((rc = ln_gemm(KT_GC_LN, w.hid_m, g2m_mesh, Nm, vm0_f32, w.vm, w.vm_img, nullptr, st))) return rc;
      if ((rc = hidden<0>(KT_GC_HIDDEN, AOperand(w.vg_img, GC_NKB), L, g2m_grid.w1, g2m_grid.b1, Ng, w.hid, nullptr, 0, nullptr, nullptr, 0, nullptr, st))) return rc;
      if ((rc = ln_gemm(KT_GC_LN, w.hid, g2m_grid, Ng, nullptr, nullptr, w.vg_img, nullptr, st, w.vg_img))) return rc;
      if (stop_after == 1) continue;
      // ---------------- processor
      bool stopped = false;
      for (int i = 0; i < cfg.layers; ++i) {
        const uint8_t* em_in_img = i ? w.em_img : e_mesh_img;
        if ((rc = table(KT_GC_TABLE, w.vm_img, proc_wsr[i], Nm, w.tm, st))) return rc;
        if ((rc = hidden<2>(KT_GC_HIDDEN, AOperand(em_in_img, GC_NKB), L, proc_edge[i].w1, proc_edge[i].b1, Em, w.hid_m, w.tm, 2 * L, mesh_s, w.tm + L,
                            2 * L, mesh_r, st))) return rc;
        // the edge latents are not read after the last layer: only the update image (for the aggregation) is produced there
        const bool last = i == cfg.layers - 1 && stop_after == 99;
        if ((rc = ln_gemm(KT_GC_LN, w.hid_m, proc_edge[i], Em, nullptr, nullptr, last ? nullptr : w.em_img, w.ym_img, st,
                          last ? nullptr : em_in_img))) return rc;
        if ((rc = segsum(KT_GC_AGG, w.ym_img, mesh_seg, w.agg_img, st))) return rc;
        if ((rc = hidden<0>(KT_GC_HIDDEN, AOperand(w.vm_img, GC_NKB).add(w.agg_img, GC_NKB), 2 * L, proc_node[i].w1, proc_node[i].b1, Nm, w.hid_m, nullptr, 0, nullptr, nullptr, 0,
                            nullptr, st))) return rc;
        if ((rc = ln_gemm(KT_GC_LN, w.hid_m, proc_node[i], Nm, w.vm, w.vm, w.vm_img, nullptr, st))) return rc;
        if (stop_after == 2 + i) { stopped = true; break; }
      }
      if (stopped) continue;
      // ---------------- decoder
      if ((rc = table(KT_GC_TABLE, w.vm_img, m2g_ws, Nm, w.tm, st))) return rc;
      if ((rc = table(KT_GC_TABLE, w.vg_img, m2g_wr, Ng, w.tg, st))) return rc;
      if ((rc = hidden<2>(KT_GC_HIDDEN, AOperand(e_m2g_img, GC_NKB), L, m2g_edge.w1, m2g_edge.b1, E3, w.hid, w.tm, L, m2g_s, w.tg, L, m2g_r, st))) return rc;
      if ((rc = ln_gemm(KT_GC_LN, w.hid, m2g_edge, E3, nullptr, nullptr, nullptr, w.yimg, st))) return rc;
      {
        const size_t seg = img_bytes(Ngp, GC_NKB);
        const AOperand a = AOperand(w.vg_img, GC_NKB).add(w.yimg, GC_NKB).add(w.yimg + seg, GC_NKB).add(w.yimg + 2 * seg, GC_NKB);
        if ((rc = hidden<0>(KT_GC_HIDDEN, a, 4 * L, m2g_grid.w1, m2g_grid.b1, Ng, w.hid, nullptr, 0, nullptr, nullptr, 0, nullptr, st))) return rc;
      }
      if ((rc = ln_gemm(KT_GC_LN, w.hid, m2g_grid, Ng, nullptr, nullptr, w.vg_img, nullptr, st, w.vg_img))) return rc;
      if ((rc = range_scan(0, w.feat, img_bytes(Ng, GC_FEAT_KP / 64), st))) return rc;
      if (stop_after == 100) continue;
      if ((rc = hidden<0>(KT_GC_HIDDEN, AOperand(w.vg_img, GC_NKB), L, out_mlp.w1, out_mlp.b1, Ng, w.hid, nullptr, 0, nullptr, nullptr, 0, nullptr, st))) return rc;
      {
        EpiGcOut epi{};
        epi.xout = xo + (size_t)cfg.n_state * plane; epi.xin = xi + (size_t)cfg.n_state * plane;
        epi.bias = out_mlp.b2; epi.dstd = dstd; epi.plane = plane; epi.nprog = cfg.n_prog;
        prof_begin(KT_GC_OUT, st);
        count_launch();
        rc = launch_gemm2<128>(SchedW<>{AOperand(w.hid, GC_NKB), out_mlp.w2.img, L / 64}, epi, Ng, 128, 1, num_sms, st);
        prof_end(KT_GC_OUT, st);
        if (rc) return rc;
      }
    }
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }

  int debug_copy(const char* what, float* dst, uint64_t max_floats, void* ws_base, int, cudaStream_t st) override {
    const Ws w = carve(ws_base);
    const float* src = nullptr; uint64_t n = 0;
    if (!strcmp(what, "range")) { src = range_dev; n = 8; if (!src) { set_error("range guard was never enabled"); return SKY_ERR_STATE; } }
    else if (!strcmp(what, "vm")) { src = w.vm; n = (uint64_t)Nm * GC_L; }
    else if (!strcmp(what, "vm0")) { src = vm0_f32; n = (uint64_t)Nm * GC_L; }
    else if (!strcmp(what, "vg") || !strcmp(what, "em") || !strcmp(what, "e_mesh")) {
      // grid-node and mesh-edge latents exist only as fp16 operand images
      const uint8_t* im = what[0] == 'v' ? w.vg_img : !strcmp(what, "em") ? w.em_img : e_mesh_img;
      const long long rows = what[0] == 'v' ? Ng : Em;
      if ((uint64_t)rows * GC_L > max_floats) { set_error("debug tensor '%s' needs %lld floats", what, rows * GC_L); return SKY_ERR_ARG; }
      k_gc_img_to_rows<<<(unsigned)((rows * (GC_L / 8) + 255) / 256), 256, 0, st>>>(im, dst, rows);
      SKY_CUDA_OK(cudaGetLastError());
      return 0;
    }
    else { set_error("unknown debug tensor '%s'", what); return SKY_ERR_ARG; }
    if (n > max_floats) { set_error("debug tensor '%s' needs %llu floats", what, (unsigned long long)n); return SKY_ERR_ARG; }
    SKY_CUDA_OK(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
};

Engine* make_graphcast_engine(const sky_graphcast_config_t& cfg, int device) {
  if (cfg.nlat < 2 || cfg.nlon < 8 || cfg.n_mesh <= 0 || cfg.n_mesh_edges <= 0 || cfg.n_g2m_edges <= 0 || cfg.layers <= 0) {
    set_error("bad GraphCast configuration");
    return nullptr;
  }
  return new GraphCastEngine(cfg, device);
}

int toa_radiation_launch(float* out, int nlat, int nlon, double unix_seconds, cudaStream_t st) {
  const long long n = (long long)nlat * nlon;
  k_gc_toa<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(out, nlat, nlon, unix_seconds);
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sky
