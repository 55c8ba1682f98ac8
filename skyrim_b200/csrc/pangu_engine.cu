// Pangu-Weather 6-h step operator on sm_90a: weight repacking + the per-step kernel
// sequence.  Replaces the two ONNX Runtime sessions that Skyrim's Pangu model
// (skyrim/core/models/pangu.py) loads and steps.
//
// Data flow (v2): every token matrix lives in NATURAL token order (member, z, lat, lon).
//   x   fp32 row-major (rows, C)                  the residual stream
//   xh  fp16 "tile image" [rows/128][C/64][128x128B SWIZZLE_128B]   = the A operand of the next
//       GEMM, written by the epilogue that produced x and fetched by 1-D bulk copies
// Windowing / cyclic shift / padding exist only as index arithmetic inside the attention kernel.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "attention_tc.cuh"
#include "engine.h"
#include "gemm2.cuh"
#include "gemm_tc.cuh"
#ifdef SKY_EXPERIMENTS
// development build only (libskyrim_b200_dev.so): CUDA-core reference GEMMs under the same epilogues, the single-CTA
// kernel variants and the result-invalidating timing switches.  None of this is compiled into the product library.
#include "gemm2_ref.cuh"
#include "gemm_ref.cuh"
#endif

namespace sky {

// ======================================================================================
// weight repacking (runs once, at load)
// ======================================================================================
// fp32 W (logical [Nsrc, K]; stored [Nsrc,K] or, if transposed, [K,Nsrc]) -> rows
// [n_off, n_off+Nsrc) of   plain fp16 [Ntot, Kp]   and   tile image
// [Ntot/BN][Kp/64][BN rows x 128 B, SWIZZLE_128B]
__global__ void k_pack_weight(const float* __restrict__ W, int Nsrc, int K, int Kp, int BN, int transposed,
                              int n_off, __half* __restrict__ plain, uint8_t* __restrict__ img) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one 8-half chunk each
  int chunks_per_row = Kp / 8;
  if (idx >= (long long)Nsrc * chunks_per_row) return;
  int ns = (int)(idx / chunks_per_row), kc = (int)(idx % chunks_per_row);
  __half h[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    int k = kc * 8 + e;
    float v = 0.f;
    if (k < K) v = transposed ? W[(long long)k * Nsrc + ns] : W[(long long)ns * K + k];
    h[e] = __float2half_rn(v);
  }
  uint4 pk = *reinterpret_cast<uint4*>(h);
  const int n = n_off + ns;
  *reinterpret_cast<uint4*>(plain + (long long)n * Kp + kc * 8) = pk;
  int nt = n / BN, nr = n % BN, kb = kc / 8, ch = kc % 8;
  size_t tile = ((size_t)nt * (Kp / 64) + kb) * (size_t)BN * 128;
  *reinterpret_cast<uint4*>(img + tile + sw128_offset(nr, ch)) = pk;
}

// earth-specific bias (3312, n_type, heads) -> (n_type, heads, 3312), pre-scaled by log2(e)
// (the attention kernel computes its softmax with exp2)
__global__ void k_pack_bias_table(const float* __restrict__ src, __half* __restrict__ dst, int L, int n_type,
                                  int heads) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long tot = (long long)L * n_type * heads;
  if (idx >= tot) return;
  int l = (int)(idx % L);
  long long th = idx / L;  // type*heads + head
  dst[idx] = __float2half_rn(src[(long long)l * n_type * heads + th] * 1.4426950408889634f);
}

// DownSample front end: 2x2 (lat, lon) merge + zero pad + LayerNorm(4C) -> fp16 tile image.
// One warp per output row; NPL = (4C)/32 values per lane.
template <int NPL>
__global__ void __launch_bounds__(256) k_down_merge_ln(const float* __restrict__ x, const uint8_t* __restrict__ ximg, uint8_t* __restrict__ img,
                                                       const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float eps, int H, int W,
                                                       int C, int H2, int W2, long long rows) {
  long long row = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  int lane = threadIdx.x % 32;
  if (row >= rows) return;
  int w2 = (int)(row % W2); long long q = row / W2;
  int h2 = (int)(q % H2); q /= H2;  // q = member*Z + z
  // lane owns 4 consecutive features per 128-feature slab: 128-bit loads, 64-bit image stores
  static_assert(NPL % 4 == 0, "features per lane");
  float v[NPL];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NPL / 4; ++i) {
    const int e = 4 * lane + 128 * i;  // feature index in (hs, ws, c); C % 4 == 0, so the four share (hs, ws)
    const int sub = e / C, c = e % C;
    const int h = 2 * h2 + (sub >> 1), w = 2 * w2 + (sub & 1);
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (h < H) {
      const long long src = (q * H + h) * W + w;
      if (ximg) {   // the token stream exists only as its fp16 operand image: 4 features = 8 bytes
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(ximg + img_offset(src, c, C / 64)));
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b2 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        t = make_float4(a.x, a.y, b2.x, b2.y);
      } else {
        t = __ldg(reinterpret_cast<const float4*>(x + src * C + c));
      }
    }
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    s += (t.x + t.y) + (t.z + t.w);
  }
  float mean = warp_sum(s) / (NPL * 32);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NPL; ++i) { float d = v[i] - mean; ss += d * d; }
  float rstd = rsqrtf(warp_sum(ss) / (NPL * 32) + eps);
#pragma unroll
  for (int i = 0; i < NPL / 4; ++i) {
    const int e = 4 * lane + 128 * i;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + e)), b = __ldg(reinterpret_cast<const float4*>(beta + e));
    uint2 pk;
    pk.x = pack_half2((v[4 * i] - mean) * rstd * g.x + b.x, (v[4 * i + 1] - mean) * rstd * g.y + b.y);
    pk.y = pack_half2((v[4 * i + 2] - mean) * rstd * g.z + b.z, (v[4 * i + 3] - mean) * rstd * g.w + b.w);
    *reinterpret_cast<uint2*>(img + img_offset(row, e, NPL / 2)) = pk;
  }
}

// test tap: fp16 image -> fp32 row-major
__global__ void k_image_to_rows(const uint8_t* __restrict__ img, int nkb, float* __restrict__ out, long long rows,
                                int cols) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  long long r = idx / cols; int c = (int)(idx % cols);
  out[idx] = __half2float(*reinterpret_cast<const __half*>(img + img_offset(r, c, nkb)));
}

// ======================================================================================
// engine
// ======================================================================================
struct GemmW {
  uint8_t* img = nullptr;
  __half* plain = nullptr;
  int N = 0, K = 0, Kp = 0, BN = 0;
};
struct BlockW {
  GemmW qkv, proj, fc1, fc2;
  GemmW proj_s, fc2_s;  // C = 384: projection and fc2 packed in 192-row halves for the column-split pair kernel (k_gemm2_pair)
  const float *qkv_b, *proj_b, *fc1_b, *fc2_b, *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  __half* bias_tab;  // (n_type, heads, 3312), fp16, pre-scaled by log2 e
};

struct PanguEngine : Engine {
  sky_pangu_config_t cfg;
  Geo g1, g2;
  int nch, nup;
  bool use_ref = false;
  // Token stream storage (sky_model_debug_set "fp32_stream"): true = only the fp16 operand image (default: 8 of the 12 bytes
  // per token and feature of the projection / MLP epilogues disappear; step error 5.8e-4 instead of 5.1e-4 at 721x1440),
  // false = fp32 rows beside the image (round-1 / early round-2 data flow; for weights whose error margin is tighter)
  bool img_stream = true;
  bool proj_split = true;   // C = 384 LayerNorm GEMMs (projection, fc2) on column-split CTA pairs ("proj_split" 0: one 384-column tile)
  int exp_qkv = 0, exp_ln = 0;  // dev build only: result-invalidating timing experiments
  bool attn_ref = false;        // dev build only (SKY_ATTN=ref): CUDA-core reference attention on the same window image
  std::vector<void*> owned;
  GemmW embed_u, embed_s, down, up1, up2, rec;
  std::vector<BlockW> blocks[4];
  const float *mean, *stdv, *masks, *embed_u_b, *embed_s_b, *down_g, *down_b, *up_g, *up_b;
  float* rec_b = nullptr;  // 5 upper + 4 surface

  PanguEngine(const sky_pangu_config_t& c, int dev) : cfg(c) {
    device = dev;
    nup = 5 * c.n_levels;
    nch = nup + 4;
    auto mk = [&](int H, int W, int C, int heads) {
      Geo g;
      g.Z = (c.n_levels + 1) / 2 + 1;
      g.H = H; g.W = W; g.C = C;
      g.Hp = (H + WH - 1) / WH * WH;
      g.nWz = g.Z / WZ; g.nWh = g.Hp / WH; g.nWw = W / WW;
      g.T = g.Z * H * W; g.nWin = g.nWz * g.nWh * g.nWw; g.heads = heads;
      return g;
    };
    int H = (c.nlat + 3) / 4, W = c.nlon / 4;
    g1 = mk(H, W, c.dim, c.heads[0]);
    g2 = mk((H + 1) / 2, W / 2, 2 * c.dim, c.heads[1]);
#ifdef SKY_EXPERIMENTS   // read once, at creation; the product library reads no environment variable at all
    const char* e = getenv("SKY_GEMM");
    use_ref = e && !strcmp(e, "ref");
    exp_qkv = getenv("SKY_QKV_EXP") ? atoi(getenv("SKY_QKV_EXP")) : 0;
    exp_ln = getenv("SKY_LN_EXP") ? atoi(getenv("SKY_LN_EXP")) : 0;
    const char* at = getenv("SKY_ATTN");
    attn_ref = at && !strcmp(at, "ref");
#endif
  }
  ~PanguEngine() override {
    for (void* p : owned) cudaFree(p);
  }

  template <class T>
  T* dalloc(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n * sizeof(T)) != cudaSuccess) { set_error("cudaMalloc(%zu) failed", n * sizeof(T)); return nullptr; }
    owned.push_back(p);
    return reinterpret_cast<T*>(p);
  }

  int pack_alloc(GemmW& g, int N, int K, int BN) {
    g.N = N; g.K = K; g.Kp = (K + 63) / 64 * 64; g.BN = BN;
    if (N % BN) { set_error("N=%d not a multiple of BLOCK_N=%d", N, BN); return SKY_ERR_ARG; }
    g.plain = dalloc<__half>((size_t)N * g.Kp);
    g.img = dalloc<uint8_t>((size_t)N * g.Kp * 2);
    return (g.plain && g.img) ? 0 : SKY_ERR_NOMEM;
  }
  int pack_rows(GemmW& g, const char* name, int Nsrc, int n_off, bool transposed, cudaStream_t st) {
    const float* w = param(name, (uint64_t)Nsrc * g.K);
    if (!w) return SKY_ERR_ARG;
    long long chunks = (long long)Nsrc * g.Kp / 8;
    k_pack_weight<<<(unsigned)((chunks + 255) / 256), 256, 0, st>>>(w, Nsrc, g.K, g.Kp, g.BN, transposed ? 1 : 0, n_off,
                                                                 g.plain, g.img);
    count_launch();
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }
  int pack(GemmW& g, const char* name, int N, int K, int BN, bool transposed, cudaStream_t st) {
    int rc = pack_alloc(g, N, K, BN);
    return rc ? rc : pack_rows(g, name, N, 0, transposed, st);
  }

  int prepare(cudaStream_t st) override {
    const int C = cfg.dim;
#define P(dst, name, cnt) if (!((dst) = keep(name, (uint64_t)(cnt), st))) return SKY_ERR_ARG;   // persistent copies
    P(mean, "norm.mean", nch); P(stdv, "norm.std", nch);
    P(masks, "const.masks", 3LL * cfg.nlat * cfg.nlon);
    P(embed_u_b, "embed.upper.b", C); P(embed_s_b, "embed.surf.b", C);
    P(down_g, "down.ln.g", 4 * C); P(down_b, "down.ln.b", 4 * C);
    P(up_g, "up.ln.g", C); P(up_b, "up.ln.b", C);
    const float *ru = param("recover.upper.b", 5), *rs = param("recover.surf.b", 4);
    if (!ru || !rs) return SKY_ERR_ARG;
    rec_b = dalloc<float>(16);
    if (!rec_b) return SKY_ERR_NOMEM;
    SKY_CUDA_OK(cudaMemcpyAsync(rec_b, ru, 5 * 4, cudaMemcpyDeviceToDevice, st));
    SKY_CUDA_OK(cudaMemcpyAsync(rec_b + 5, rs, 4 * 4, cudaMemcpyDeviceToDevice, st));
    int rc;
    if ((rc = pack(embed_u, "embed.upper.w", C, 160, 192, false, st))) return rc;
    if ((rc = pack(embed_s, "embed.surf.w", C, 112, 192, false, st))) return rc;
    if ((rc = pack(down, "down.w", 2 * C, 4 * C, 192, false, st))) return rc;
    if ((rc = pack(up1, "up.w1", 4 * C, 2 * C, 192, false, st))) return rc;
    if ((rc = pack(up2, "up.w2", C, C, 192, false, st))) return rc;
    // patch recovery: one N = 160 + 64 weight (upper-air | surface columns)
    if ((rc = pack_alloc(rec, 224, 2 * C, 224))) return rc;
    if ((rc = pack_rows(rec, "recover.upper.w", 160, 0, true, st))) return rc;
    if ((rc = pack_rows(rec, "recover.surf.w", 64, 160, true, st))) return rc;
    for (int li = 0; li < 4; ++li) {
      const Geo& g = (li == 0 || li == 3) ? g1 : g2;
      const int c = g.C, heads = cfg.heads[li], n_type = g.nWz * g.nWh;
      blocks[li].resize(cfg.depths[li]);
      for (int bi = 0; bi < cfg.depths[li]; ++bi) {
        BlockW& b = blocks[li][bi];
        char nm[96];
        auto N = [&](const char* s) { snprintf(nm, sizeof nm, "layer%d.block%d.%s", li, bi, s); return nm; };
        if ((rc = pack(b.qkv, N("qkv.w"), 3 * c, c, 192, false, st))) return rc;
        if ((rc = pack(b.proj, N("proj.w"), c, c, c, false, st))) return rc;
        if (c == 384 && (rc = pack(b.proj_s, N("proj.w"), c, c, 192, false, st))) return rc;
        if ((rc = pack(b.fc1, N("fc1.w"), 4 * c, c, 192, false, st))) return rc;
        if ((rc = pack(b.fc2, N("fc2.w"), c, 4 * c, c, false, st))) return rc;
        if (c == 384 && (rc = pack(b.fc2_s, N("fc2.w"), c, 4 * c, 192, false, st))) return rc;
        P(b.qkv_b, N("qkv.b"), 3 * c); P(b.proj_b, N("proj.b"), c);
        P(b.fc1_b, N("fc1.b"), 4 * c); P(b.fc2_b, N("fc2.b"), c);
        P(b.ln1_g, N("ln1.g"), c); P(b.ln1_b, N("ln1.b"), c);
        P(b.ln2_g, N("ln2.g"), c); P(b.ln2_b, N("ln2.b"), c);
        long long tot = (long long)AT_TABLE * n_type * heads;
        const float* bt = param(N("bias_table"), (uint64_t)tot);   // transient: repacked below
        if (!bt) return SKY_ERR_ARG;
        b.bias_tab = dalloc<__half>((size_t)tot);
        if (!b.bias_tab) return SKY_ERR_NOMEM;
        k_pack_bias_table<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(bt, b.bias_tab, AT_TABLE, n_type, heads);
        count_launch();
      }
    }
#undef P
    SKY_CUDA_OK(cudaGetLastError());
    SKY_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  }

  // ---- workspace carving -----------------------------------------------------------------
  struct Ws {
    float *x1, *x2, *scratch;
    uint8_t *x1h, *skiph, *x2h, *atth, *hidh;
    uint8_t* qkv;
    size_t x1h_bytes;
    size_t total;
  };
  static size_t tiles(long long rows) { return (size_t)((rows + 127) / 128); }
  Ws carve(void* base, int B) const {
    Ws w;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 1023) / 1024 * 1024; return (char*)base + o; };
    const size_t C = cfg.dim;
    const long long R1 = (long long)B * g1.T, R2 = (long long)B * g2.T;
    const size_t t1 = tiles(R1), t2 = tiles(R2);
    w.x1 = (float*)take((size_t)R1 * C * 4);
    w.x2 = (float*)take((size_t)R2 * 2 * C * 4);
    w.x1h_bytes = t1 * (C / 64) * G2_A_BYTES;
    w.x1h = (uint8_t*)take(w.x1h_bytes);
    w.skiph = (uint8_t*)take(w.x1h_bytes);
    w.x2h = (uint8_t*)take(t2 * (2 * C / 64) * G2_A_BYTES);
    // q | k | v window images (attention_tc.cuh): one 144-row x 128-byte tile per (member, window, head pair) and part
    const size_t wt1 = (size_t)B * g1.nWin * (g1.heads / 2), wt2 = (size_t)B * g2.nWin * (g2.heads / 2);
    w.qkv = (uint8_t*)take(3 * (wt1 > wt2 ? wt1 : wt2) * AT_TILE_B);
    size_t att_b = t1 * (C / 64) > t2 * (2 * C / 64) ? t1 * (C / 64) : t2 * (2 * C / 64);
    w.atth = (uint8_t*)take(att_b * G2_A_BYTES);
    size_t hid_b = t1 * (4 * C / 64) > t2 * (8 * C / 64) ? t1 * (4 * C / 64) : t2 * (8 * C / 64);
    w.hidh = (uint8_t*)take(hid_b * G2_A_BYTES);  // MLP hidden; also the down-sample / up-sample staging images
    size_t scr = 0;
    if (use_ref) scr = (size_t)R1 * 4 * C * 4;
    w.scratch = (float*)take(scr);
    w.total = off;
    return w;
  }
  size_t workspace_bytes(int batch) const override { return carve(nullptr, batch).total; }

  // ---- GEMM dispatch -----------------------------------------------------------------------
  template <int BN, class Epi>
  int gemm2(int tag, const AOperand& A, const Epi& epi, const GemmW& w, long long M, float* scratch, cudaStream_t st) {
    if (w.BN != BN) { set_error("internal: weight packed for BLOCK_N=%d used with %d", w.BN, BN); return SKY_ERR_STATE; }
    int rc;
    prof_begin(tag, st);
#ifdef SKY_EXPERIMENTS
    if (use_ref) {
      count_launch(2);
      rc = launch_gemm2_ref<Epi, BN>(A, epi, w.plain, scratch, M, w.N, w.Kp, st);
    } else
#endif
    {
      count_launch();
      rc = launch_gemm2<BN>(SchedW<>{A, w.img, w.Kp / 64}, epi, M, w.N, 1, num_sms, st);
    }
    prof_end(tag, st);
    return rc;
  }
  // patch embedding keeps warp producers (im2col + normalisation of the fp32 state)
  template <int BN, class Prod, class Epi>
  int gemm_prod(int tag, const Prod& prod, const Epi& epi, const GemmW& w, long long M, float* scratch, cudaStream_t st) {
    int rc;
    prof_begin(tag, st);
#ifdef SKY_EXPERIMENTS
    if (use_ref) {
      count_launch(2);
      rc = launch_gemm_ref(prod, epi, w.plain, scratch, M, w.N, w.Kp, BN, st);
    } else
#endif
    {
      count_launch();
      rc = launch_gemm_tc<Prod, Epi, BN>(prod, epi, w.img, M, w.N, w.Kp, num_sms, st);
    }
    prof_end(tag, st);
    return rc;
  }

  // IMG: the token stream of this handle lives only as its fp16 operand image (img_stream) — the LayerNorm epilogues then read
  // the residual from xh and write xh in place; otherwise x (fp32 rows) is read-modify-written beside the image.
  int run_block(float* x, uint8_t* xh, const Geo& g, const BlockW& b, int roll, int B, const Ws& ws, cudaStream_t st) {
    return img_stream ? run_block_t<true>(x, xh, g, b, roll, B, ws, st) : run_block_t<false>(x, xh, g, b, roll, B, ws, st);
  }
  template <bool IMG>
  int run_block_t(float* x, uint8_t* xh, const Geo& g, const BlockW& b, int roll, int B, const Ws& ws, cudaStream_t st) {
    using ELn = Epi2F32Img<true, true, IMG>;
    const int C = g.C, nkb = C / 64;
    const long long R = (long long)B * g.T;
    int rc;
    const int pairs = g.heads / 2;
    const long long part_stride = (long long)B * g.nWin * pairs * AT_TILE_B;
    {  // QKV projection: natural-order tokens in, window image out (windowing / shift / padding applied by the epilogue)
      AOperand A(xh, nkb);
      EpiQkvWin e{ws.qkv, part_stride, b.qkv_b, g, roll, C, pairs};
#ifdef SKY_EXPERIMENTS
      e.exp = exp_qkv;
#endif
      if ((rc = gemm2<192>(KT_QKV, A, e, b.qkv, R, ws.scratch, st))) return rc;
      if (g.Hp > g.H) {   // latitude-padding tokens (x = 0): their q, k, v rows are the projection's bias.  (Writing them from
                          // the GEMM epilogue of the neighbouring tokens instead cost the GEMM 0.5 ms/step: measured, reverted.)
        const long long total = 3LL * B * g.Z * (g.Hp - g.H) * g.W * pairs * 8;
        prof_begin(KT_QKV, st);
        k_qkv_fill_pad<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ws.qkv, part_stride, b.qkv_b, g, roll, B, pairs, C, total);
        prof_end(KT_QKV, st);
        count_launch();
        SKY_CUDA_OK(cudaGetLastError());
      }
    }
    {
      AttnArgs a{ws.qkv, part_stride, ws.atth, nkb, b.bias_tab, g, roll, B, pairs,
                 rsqrtf(32.f) * 1.4426950408889634f, cfg.mask_value * 1.4426950408889634f, (long long)B * g.nWin * pairs};
      prof_begin(KT_ATTN, st);
      count_launch();
#ifdef SKY_EXPERIMENTS
      if (attn_ref) {
        k_window_attention_ref<<<dim3((unsigned)a.items, 2), WIN_TOK, 0, st>>>(a);
        rc = cudaGetLastError() == cudaSuccess ? 0 : SKY_ERR_CUDA;
      } else
#endif
        rc = launch_window_attention_tc(a, num_sms, st);
      prof_end(KT_ATTN, st);
      if (rc) return rc;
    }
    {  // projection + LayerNorm + residual
      AOperand A(ws.atth, nkb);
      ELn e{x, C, xh, nkb, b.proj_b, b.ln1_g, b.ln1_b, cfg.ln_eps};
#ifdef SKY_EXPERIMENTS
      e.exp = exp_ln;
#endif
      if (C == 384 && proj_split && !use_ref) {
        // a 128 x 384 accumulator takes 192 registers per consumer thread: the two CTAs of a cluster take 192 columns each of
        // the same 128 rows, LayerNorm statistics cross through DSMEM
        prof_begin(KT_PROJ, st);
        count_launch();
        rc = launch_gemm2<192, true>(SchedW<>{A, b.proj_s.img, C / 64}, e, R, C, 1, num_sms, st);
        prof_end(KT_PROJ, st);
      } else {
        rc = C == 192 ? gemm2<192>(KT_PROJ, A, e, b.proj, R, ws.scratch, st)
                      : gemm2<384>(KT_PROJ, A, e, b.proj, R, ws.scratch, st);
      }
      if (rc) return rc;
    }
    {  // MLP: fc1 + GELU into the fp16 hidden image, then fc2 + LayerNorm + residual
      AOperand A(xh, nkb);
      Epi2F16<true, true> e{reinterpret_cast<__half*>(ws.hidh), 0, 4 * nkb, b.fc1_b};
      if ((rc = gemm2<192>(KT_FC1, A, e, b.fc1, R, ws.scratch, st))) return rc;
      AOperand A2(ws.hidh, 4 * nkb);
      ELn e2{x, C, xh, nkb, b.fc2_b, b.ln2_g, b.ln2_b, cfg.ln_eps};
#ifdef SKY_EXPERIMENTS
      e2.exp = exp_ln;
#endif
      if (C == 384 && proj_split && !use_ref) {
        prof_begin(KT_FC2, st);
        count_launch();
        rc = launch_gemm2<192, true>(SchedW<>{A2, b.fc2_s.img, 4 * C / 64}, e2, R, C, 1, num_sms, st);
        prof_end(KT_FC2, st);
      } else {
        rc = C == 192 ? gemm2<192>(KT_FC2, A2, e2, b.fc2, R, ws.scratch, st)
                      : gemm2<384>(KT_FC2, A2, e2, b.fc2, R, ws.scratch, st);
      }
      if (rc) return rc;
    }
    if (range_guard) {   // fp16 operand images of this block (whole tiles only: the tail rows of the last tile are never written)
      const size_t full = (size_t)(R / 128) * nkb * G2_A_BYTES;
      if ((rc = range_scan(0, xh, full, st))) return rc;
      if ((rc = range_scan(1, ws.qkv, (size_t)3 * part_stride, st))) return rc;
      if ((rc = range_scan(2, ws.atth, full, st))) return rc;
    }
    return 0;
  }

  int step(const float* x_in, float* x_out, int B, void* wsp, size_t ws_bytes, cudaStream_t st) override {
    if (!loaded) { set_error("weights not loaded"); return SKY_ERR_STATE; }
    Ws ws = carve(wsp, B);
    if (ws_bytes < ws.total) { set_error("workspace too small: %zu < %zu", ws_bytes, ws.total); return SKY_ERR_ARG; }
    const int C = cfg.dim, HW = g1.H * g1.W, nzt = g1.Z - 1;
    const long long R1 = (long long)B * g1.T, R2 = (long long)B * g2.T;
    int rc;
    // test tap (sky_model_debug_set "stop_after"): return early so that debug_copy can read the token buffers
    // (0 embed, 1 layer0, 2 down, 3 layer1, 4 layer2, 5 up, 6 layer3; default 99 = whole step)
    const int stop = stop_after;
    // ---- patch embedding ----
    {
      long long M = (long long)B * nzt * HW;
      ProdEmbedUpper p{x_in, mean, stdv, cfg.nlat, cfg.nlon, cfg.n_levels, 5, nch, g1.H, g1.W, nzt, M};
      EpiStoreF32 e{img_stream ? nullptr : ws.x1, C, embed_u_b, M, g1.T, HW, 1, (long long)nzt * HW, ws.skiph, C / 64};
      if ((rc = gemm_prod<192>(KT_EMBED, p, e, embed_u, M, ws.scratch, st))) return rc;
      long long Ms = (long long)B * HW;
      ProdEmbedSurf ps{x_in, masks, mean, stdv, cfg.nlat, cfg.nlon, nch, nup, 4, 3, g1.H, g1.W, Ms};
      EpiStoreF32 es{img_stream ? nullptr : ws.x1, C, embed_s_b, Ms, g1.T, HW, 0, (long long)HW, ws.skiph, C / 64};
      if ((rc = gemm_prod<192>(KT_EMBED, ps, es, embed_s, Ms, ws.scratch, st))) return rc;
    }
    if (stop == 0) return 0;
    for (size_t i = 0; i < blocks[0].size(); ++i)
      if ((rc = run_block(ws.x1, ws.skiph, g1, blocks[0][i], (int)(i & 1), B, ws, st))) return rc;
    if (stop == 1) return 0;
    // the first layer works in place on the skip image: its final operand image IS the skip connection that patch
    // recovery concatenates, the up-sample path writes the other image (x1h) — no copy
    // ---- down-sample ----
    {
      prof_begin(KT_DOWN, st);
      k_down_merge_ln<24><<<(unsigned)((R2 + 7) / 8), 256, 0, st>>>(ws.x1, img_stream ? ws.skiph : nullptr, ws.hidh, down_g, down_b,
                                                                 cfg.ln_eps, g1.H, g1.W, C, g2.H, g2.W, R2);
      prof_end(KT_DOWN, st);
      count_launch();
      SKY_CUDA_OK(cudaGetLastError());
      AOperand A(ws.hidh, 4 * C / 64);
      if (img_stream) {
        Epi2F32Img<false, false, true> e{ws.x2, 2 * C, ws.x2h, 2 * C / 64, nullptr, nullptr, nullptr, 0.f};
        rc = gemm2<192>(KT_DOWN, A, e, down, R2, ws.scratch, st);
      } else {
        Epi2F32Img<false, false, false> e{ws.x2, 2 * C, ws.x2h, 2 * C / 64, nullptr, nullptr, nullptr, 0.f};
        rc = gemm2<192>(KT_DOWN, A, e, down, R2, ws.scratch, st);
      }
      if (rc) return rc;
      if ((rc = range_scan(3, ws.x2h, (size_t)(R2 / 128) * (2 * C / 64) * G2_A_BYTES, st))) return rc;
    }
    if (stop == 2) return 0;
    for (int li = 1; li <= 2; ++li) {
      for (size_t i = 0; i < blocks[li].size(); ++i)
        if ((rc = run_block(ws.x2, ws.x2h, g2, blocks[li][i], (int)(i & 1), B, ws, st))) return rc;
      if (stop == 2 + li) return 0;
    }
    // ---- up-sample ----
    {
      AOperand A(ws.x2h, 2 * C / 64);
      Epi2UpShuffle e{ws.hidh, C / 64, C, up_g, up_b, cfg.ln_eps, nullptr, g1.H, g1.W, g2.H, g2.W};
      if ((rc = gemm2<192>(KT_UP, A, e, up1, R2, ws.scratch, st))) return rc;
      AOperand A2(ws.hidh, C / 64);
      if (img_stream) {
        Epi2F32Img<false, false, true> e2{ws.x1, C, ws.x1h, C / 64, nullptr, nullptr, nullptr, 0.f};
        rc = gemm2<192>(KT_UP, A2, e2, up2, R1, ws.scratch, st);
      } else {
        Epi2F32Img<false, false, false> e2{ws.x1, C, ws.x1h, C / 64, nullptr, nullptr, nullptr, 0.f};
        rc = gemm2<192>(KT_UP, A2, e2, up2, R1, ws.scratch, st);
      }
      if (rc) return rc;
    }
    if (stop == 5) return 0;
    for (size_t i = 0; i < blocks[3].size(); ++i)
      if ((rc = run_block(ws.x1, ws.x1h, g1, blocks[3][i], (int)(i & 1), B, ws, st))) return rc;
    if (stop == 6) return 0;
    // ---- patch recovery: concat(skip, x) along K, one GEMM for upper-air + surface ----
    {
      const AOperand A = AOperand(ws.skiph, C / 64).add(ws.x1h, C / 64);
      Epi2Recover e{x_out, rec_b, mean, stdv, cfg.nlat, cfg.nlon, nch, nup, cfg.n_levels, g1.H, g1.W, g1.T};
      if ((rc = gemm2<224>(KT_RECOVER, A, e, rec, R1, ws.scratch, st))) return rc;
    }
    return 0;
  }

  int debug_set(const char* key, long long value) override {
    if (!strcmp(key, "fp32_stream")) { img_stream = value == 0; drop_graphs(); return 0; }
    if (!strcmp(key, "proj_split")) { proj_split = value != 0; drop_graphs(); return 0; }
    return Engine::debug_set(key, value);
  }

  int debug_copy(const char* what, float* dst, uint64_t max_floats, void* wsp, int B, cudaStream_t st) override {
    Ws ws = carve(wsp, B);
    const float* src = nullptr;
    uint64_t n = 0;
    const long long R1 = (long long)B * g1.T, R2 = (long long)B * g2.T;
    const bool stream_tap = img_stream && (!strcmp(what, "tokens1") || !strcmp(what, "tokens2"));
    if (!stream_tap && !strcmp(what, "tokens1")) { src = ws.x1; n = (uint64_t)R1 * cfg.dim; }
    else if (!stream_tap && !strcmp(what, "tokens2")) { src = ws.x2; n = (uint64_t)R2 * 2 * cfg.dim; }
    else if (stream_tap || !strcmp(what, "tokens1_h") || !strcmp(what, "tokens2_h") || !strcmp(what, "skip_h")) {
      // the fp16 operand image, expanded to fp32 rows.  With the image-only token stream "tokens1" is the skip image until the
      // down-sample (embedding and first layer work in place on it) and the x1 image from the up-sample on.
      const bool two = what[6] == '2';
      const uint8_t* img = two ? ws.x2h : ((!strcmp(what, "skip_h") || (stream_tap && stop_after <= 1)) ? ws.skiph : ws.x1h);
      const long long rows = two ? R2 : R1;
      const int cols = two ? 2 * cfg.dim : cfg.dim;
      if ((uint64_t)rows * cols > max_floats) { set_error("destination too small"); return SKY_ERR_ARG; }
      k_image_to_rows<<<(unsigned)((rows * cols + 255) / 256), 256, 0, st>>>(img, cols / 64, dst, rows, cols);
      SKY_CUDA_OK(cudaGetLastError());
      return 0;
    } else if (!strcmp(what, "range")) {
      if (!range_dev || max_floats < 8) { set_error("range guard is off (debug_set range_guard 1) or destination < 8 floats"); return SKY_ERR_STATE; }
      src = range_dev; n = 8;
    } else { set_error("unknown debug buffer '%s'", what); return SKY_ERR_ARG; }
    if (n > max_floats) n = max_floats;
    SKY_CUDA_OK(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
};

Engine* make_pangu_engine(const sky_pangu_config_t& cfg, int device) {
  if (cfg.nlon % 96 || cfg.nlat < 8 || cfg.n_levels != 13 || cfg.dim != 192) {
    set_error("unsupported Pangu shape: nlat=%d nlon=%d (need nlon %% 96 == 0) levels=%d dim=%d", cfg.nlat, cfg.nlon,
              cfg.n_levels, cfg.dim);
    return nullptr;
  }
  for (int i = 0; i < 4; ++i) {
    int c = (i == 0 || i == 3) ? cfg.dim : 2 * cfg.dim;
    if (cfg.heads[i] * 32 != c) { set_error("head_dim must be 32"); return nullptr; }
  }
  return new PanguEngine(cfg, device);
}

}  // namespace sky
