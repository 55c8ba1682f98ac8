// Kernel-level probe of the wgmma GEMM (gemm2.cuh / gemm_tb.cuh), for tests only: libskyrim_b200_probe.so.
//
// sky_probe_gemm launches ONE k_gemm2 / k_gemm2_pair with a schedule and an epilogue built from raw device pointers,
// so that tests/test_gemm_kernels_gpu.py can compare the kernel element by element against the fp64 reference of
// oracle/gemm_ref.py at shapes the models never reach.  It is dispatch glue only: the operands arrive already packed
// (fp16 tile images built by the test), and every (schedule, epilogue, BLOCK_N) below is one the engines instantiate.
//
// The library links the engine objects, which instantiate the same kernels from the same sources and flags.  The
// linker keeps one host stub per kernel instantiation, so the probe may launch the engine object's copy of a kernel
// rather than its own: they are the same code, and a change to a kernel has to be rebuilt into all objects to show here.
//
// A case is validated on the host before anything touches the device: an inconsistent one (a k-block count that does
// not match the images, a pair launch with N != 2 BLOCK_N, ...) could read out of bounds or leave an mbarrier waiting
// forever, so it is refused with an error (sky_last_error) instead.
#include <cstdint>
#include <vector>

#include "gemm_tb.cuh"
#include "mlp_fused.cuh"
#define SKY_GC_EPILOGUES_ONLY   // graphcast_ops.cuh: the epilogues, not the engine's kernels (defined in graphcast_engine.o)
#include "graphcast_ops.cuh"
#include "attention_tc.cuh"   // EpiQkvWin (the attention kernels are defined in pangu_engine.o)
#include "probe_geo.cuh"

extern "C" {

// SKY_PROBE_MLP: Pangu's fused MLP (mlp_fused.cuh) at C = n = 192 (k_mlp_fused) or 384 (k_mlp_fused_pair), in place on the
// stream image `hi` (img_nkb = C / 64 k-blocks).  W1 at BLOCK_N 64 is `w`, W2 at BLOCK_N 192 is `b_hi` (b_bytes), the fc1 bias
// is `add` (add_bytes) and fc2's bias, gamma, beta and eps are the LayerNorm's; `epi` is ignored.
enum { SKY_PROBE_W = 0, SKY_PROBE_W_TRI = 1, SKY_PROBE_TB = 2, SKY_PROBE_PAIR = 3, SKY_PROBE_MLP = 4 };
enum {
  SKY_PROBE_EPI_F32 = 0,          // EpiF32Batched<false>
  SKY_PROBE_EPI_F32_ACC = 1,      // EpiF32Batched<true>
  SKY_PROBE_EPI_SPLIT = 2,        // EpiSplitImg<false>
  SKY_PROBE_EPI_SPLIT_GELU = 3,   // EpiSplitImg<true>
  SKY_PROBE_EPI_F32_STATS = 4,    // EpiF32ImgStats
  SKY_PROBE_EPI_GELU_STATS = 5,   // EpiGeluStatsImg
  SKY_PROBE_EPI_REMAP = 6,        // EpiSplitRemap
  SKY_PROBE_EPI_LN = 7,           // Epi2F32Img<true, 1>: fp32 rows in place, and their image
  SKY_PROBE_EPI_LN_IMG = 8,       // Epi2F32Img<true, 2>: the fp16 image in place
  SKY_PROBE_EPI_F16_GELU_IMG = 9, // Epi2F16<true, true>
  SKY_PROBE_EPI_F16_ROWS = 10,    // Epi2F16<false, false>
  SKY_PROBE_EPI_GC_SILU0 = 11,    // EpiGcSiluImg<0>
  SKY_PROBE_EPI_GC_SILU2 = 12,    // EpiGcSiluImg<2>
  SKY_PROBE_EPI_GC_OUT = 13,      // EpiGcOut
  SKY_PROBE_EPI_GC_LN0 = 14,      // Epi2F32Img<true, 0> at GraphCast's shapes
  SKY_PROBE_EPI_GC_LN1 = 15,      // Epi2F32Img<true, 1> at GraphCast's shapes
  SKY_PROBE_EPI_GC_LN2 = 16,      // Epi2F32Img<true, 2> at GraphCast's shapes
  SKY_PROBE_EPI_QKV_WIN = 17,     // FragEpi<EpiQkvWin> (Pangu's QKV projection -> q | k | v window image)
  SKY_PROBE_EPI_F16_GELU_IMG_FRAG = 18,   // FragEpi<Epi2F16<true, true>>: SKY_PROBE_EPI_F16_GELU_IMG on the fragment path
  SKY_PROBE_EPI_LN_IMG_FRAG = 19,         // FragEpi<Epi2F32Img<true, 2>>: SKY_PROBE_EPI_LN_IMG on the fragment path
};

// Every pointer is a device pointer; every *_bytes / *_floats field is the size of the allocation behind it, which the
// host-side validation checks the case's reads and writes against.
typedef struct {
  int32_t kernel, epi, block_n, n, n_valid, batches;
  int32_t grid_sms;          // passed as num_sms to launch_gemm2; 0 = the device's SM count
  int32_t nseg;              // A segments (SchedW)
  int64_t m;
  const void* a[6]; int64_t a_bytes[6]; int64_t a_batch_stride[6]; int32_t a_nkb[6];
  const void* w; int64_t w_bytes; int64_t w_batch_stride;
  int32_t num_kb, w_rep;
  // SchedTB: table [batches][M/128][hi | lo][128 x 128 B] and the MN-major data images (BData)
  const void* t; int64_t t_bytes; int64_t t_batch_stride;
  int32_t t_rows, b_nkb_img;
  const void* b_hi; const void* b_lo; int64_t b_bytes; int64_t b_rows_per_batch; int64_t b_batch_bytes;
  // epilogue
  void* out; int64_t out_bytes; int64_t out_batch_stride /*floats*/;
  int32_t ldo, img_nkb;
  void* hi; void* lo; int64_t img_bytes; int64_t img_batch_bytes;
  const float* bias; const float* gamma; const float* beta; const float* add; const float* asc; const float* ash;
  const float* csc; const float* csh; const float* t1;
  int64_t vec_floats;        // length of bias / gamma / beta / asc / ash / csc / csh
  int64_t add_bytes;
  int64_t t1_floats;
  double* sums; int64_t sums_bytes;
  int64_t rows_per_batch;    // EpiGeluStatsImg: pixel row = batch * rows_per_batch + row
  int32_t bdiv, kmul, kdiv, rb, same;
  float eps;
  // GraphCast epilogues: gathered fp16 tables ta / tb [rows][ld] indexed by ia / ib [M]; the LayerNorm's residual source
  // (xin or xin_img) and update image; EpiGcOut's channel planes
  const void* ta; const void* tb; const int32_t* ia; const int32_t* ib;
  int64_t ta_bytes, tb_bytes, ta_rows, tb_rows;
  int32_t lda, ldb;
  void* yimg; const float* xin; const void* xin_img; const float* dstd;
  int64_t xin_bytes, plane;
  int32_t nprog;
  // EpiQkvWin: the token grid (M = members x T), the cyclic shift, head pairs and the bytes between the q, k and v parts
  // of the window image `hi` (img_bytes long); the projection's bias is `bias`
  sky_probe_geo_t geo;
  int32_t roll, pairs;
  int64_t part_stride;
} sky_probe_case_t;

SKY_API int sky_probe_case_size(void) { return (int)sizeof(sky_probe_case_t); }
SKY_API int sky_probe_gemm(const sky_probe_case_t* c, void* stream);

}  // extern "C"

namespace sky {
namespace {

using Case = sky_probe_case_t;
constexpr long long TILE = G2_A_BYTES;

#define PROBE_REQUIRE(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      set_error("gemm probe: " __VA_ARGS__);     \
      return SKY_ERR_ARG;                        \
    }                                            \
  } while (0)

long long cdiv(long long a, long long b) { return (a + b - 1) / b; }
bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

// ---- host-side validation of the operands (what the loader reads) ----
int check_operands(const Case& c) {
  const long long mt = cdiv(c.m, G2_BLOCK_M);
  PROBE_REQUIRE(c.m >= 1 && c.batches >= 1 && c.n >= c.block_n && c.n % c.block_n == 0, "shape M=%lld N=%d BN=%d batches=%d",
                (long long)c.m, c.n, c.block_n, c.batches);
  PROBE_REQUIRE(c.grid_sms >= 0, "grid_sms %d", c.grid_sms);
  PROBE_REQUIRE(c.num_kb >= 1, "num_kb %d", c.num_kb);
  if (c.kernel == SKY_PROBE_TB) {
    PROBE_REQUIRE(c.n % 64 == 0, "table x data: N=%d not a multiple of 64", c.n);
    PROBE_REQUIRE(c.num_kb % 3 == 0, "table x data: num_kb=%d is not 3 x the table's k-blocks", c.num_kb);
    PROBE_REQUIRE(c.t_rows % 128 == 0 && c.m <= c.t_rows, "table x data: table rows %d (M=%lld)", c.t_rows, (long long)c.m);
    PROBE_REQUIRE(c.b_rows_per_batch % 8 == 0 && c.b_rows_per_batch >= 0, "table x data: rows_per_batch %lld not a multiple of 8",
                  (long long)c.b_rows_per_batch);
    PROBE_REQUIRE(c.b_batch_bytes % 16 == 0 && c.b_batch_bytes >= 0 && c.t_batch_stride % 16 == 0 && c.t_batch_stride >= 0,
                  "table x data: batch strides");
    PROBE_REQUIRE(c.t && c.b_hi && c.b_lo && aligned16(c.t) && aligned16(c.b_hi) && aligned16(c.b_lo), "table x data: null or misaligned operand");
    const int nkb = c.num_kb / 3;
    PROBE_REQUIRE(mt * 2 * nkb * TILE + (c.batches - 1) * c.t_batch_stride <= c.t_bytes, "table image too small");
    PROBE_REQUIRE(c.n / 64 <= c.b_nkb_img, "data image has %d column blocks, N=%d", c.b_nkb_img, c.n);
    const long long last_row = (long long)(c.batches - 1) * c.b_rows_per_batch + (long long)nkb * 64 - 1;
    PROBE_REQUIRE((c.batches - 1) * c.b_batch_bytes + (last_row / 128 + 1) * c.b_nkb_img * TILE <= c.b_bytes, "data image too small");
    return 0;
  }
  PROBE_REQUIRE(c.nseg >= 1 && c.nseg <= 6, "%d A segments (1 .. 6)", c.nseg);
  long long kb = 0;
  for (int s = 0; s < c.nseg; ++s) {
    PROBE_REQUIRE(c.a[s] && aligned16(c.a[s]) && c.a_nkb[s] >= 1 && c.a_batch_stride[s] >= 0 && c.a_batch_stride[s] % 16 == 0,
                  "A segment %d", s);
    PROBE_REQUIRE((c.batches - 1) * c.a_batch_stride[s] + mt * c.a_nkb[s] * TILE <= c.a_bytes[s], "A segment %d image too small", s);
    kb += c.a_nkb[s];
  }
  PROBE_REQUIRE(kb == c.num_kb, "A has %lld k-blocks, num_kb=%d", kb, c.num_kb);
  PROBE_REQUIRE(c.w_rep >= 0 && 2 * c.w_rep <= c.num_kb, "w_rep %d (num_kb %d)", c.w_rep, c.num_kb);
  PROBE_REQUIRE(c.w && aligned16(c.w) && c.w_batch_stride >= 0 && c.w_batch_stride % 16 == 0, "W image");
  PROBE_REQUIRE((c.batches - 1) * c.w_batch_stride + (long long)(c.n / c.block_n) * (c.num_kb - c.w_rep) * c.block_n * 128 <= c.w_bytes,
                "W image too small");
  if (c.kernel == SKY_PROBE_PAIR) {
    PROBE_REQUIRE(c.n == 2 * c.block_n && c.batches == 1, "pair: N=%d must be 2 x BN=%d, one batch", c.n, c.block_n);
    PROBE_REQUIRE(c.grid_sms == 0 || c.grid_sms >= 2, "pair: grid_sms %d < 2", c.grid_sms);
  }
  return 0;
}

// ---- host-side validation of what the epilogue writes and reads ----
int check_vec(const Case& c, const float* p, long long need, const char* what) {
  PROBE_REQUIRE(p && aligned16(p) && c.vec_floats >= need, "%s: null, misaligned or shorter than %lld", what, need);
  return 0;
}
int check_img(const Case& c, long long rows, int cols) {
  PROBE_REQUIRE(c.img_nkb >= 1 && cols <= c.img_nkb * 64, "destination image: %d k-blocks for %d columns", c.img_nkb, cols);
  PROBE_REQUIRE(cdiv(rows, G2_BLOCK_M) * c.img_nkb * TILE <= c.img_bytes, "destination image too small");
  return 0;
}
int check_split_img(const Case& c, long long rows, int cols) {
  PROBE_REQUIRE(c.hi && c.lo && aligned16(c.hi) && aligned16(c.lo), "hi / lo images");
  return check_img(c, rows, cols);
}
int check_sums(const Case& c) {
  PROBE_REQUIRE(c.n_valid <= CTA_STATS_MAX, "statistics of %d > %d channels", c.n_valid, CTA_STATS_MAX);
  PROBE_REQUIRE(!c.sums || c.sums_bytes >= 2LL * c.n_valid * 8, "sums too small");
  return 0;
}

// the gathered table rows: every index is copied to the host and checked against the table's row count
int check_gather(const Case& c, const void* t, const int32_t* idx, long long rows, int ld, long long bytes, const char* what) {
  PROBE_REQUIRE(t && idx && aligned16(t) && ld % 8 == 0 && ld >= GC_L && rows >= 1 && ((rows - 1) * ld + GC_L) * 2 <= bytes,
                "%s: table layout", what);
  std::vector<int32_t> h((size_t)c.m);
  SKY_CUDA_OK(cudaMemcpy(h.data(), idx, h.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
  for (int32_t v : h) PROBE_REQUIRE(v >= 0 && v < rows, "%s: index %d outside [0, %lld)", what, v, rows);
  return 0;
}
int check_gathers(const Case& c) {
  int rc;
  if ((rc = check_gather(c, c.ta, c.ia, c.ta_rows, c.lda, c.ta_bytes, "ta"))) return rc;
  return check_gather(c, c.tb, c.ib, c.tb_rows, c.ldb, c.tb_bytes, "tb");
}

int check_epilogue(const Case& c) {
  int rc = 0;
  PROBE_REQUIRE(c.n_valid >= 1 && c.n_valid <= c.n, "n_valid %d (N %d)", c.n_valid, c.n);
  switch (c.epi) {
    case SKY_PROBE_EPI_F32:
    case SKY_PROBE_EPI_F32_ACC: {
      // float4 stores and loads: a 4-column group is stored whole once its first column is < n_valid
      PROBE_REQUIRE(c.n_valid % 4 == 0 && c.ldo % 4 == 0 && c.ldo >= c.n_valid && c.out_batch_stride % 4 == 0, "fp32 output layout");
      const long long need = (long long)(c.batches - 1) * c.out_batch_stride + (c.m - 1) * c.ldo + c.n_valid;
      PROBE_REQUIRE(c.out && aligned16(c.out) && need * 4 <= c.out_bytes, "fp32 output too small");
      PROBE_REQUIRE(!c.add || (aligned16(c.add) && need * 4 <= c.add_bytes), "addend too small");
      if (c.bias && (rc = check_vec(c, c.bias, c.n_valid, "bias"))) return rc;
      return 0;
    }
    case SKY_PROBE_EPI_SPLIT:
    case SKY_PROBE_EPI_SPLIT_GELU:
      PROBE_REQUIRE(c.n_valid % 8 == 0, "n_valid %d: 8-column chunks", c.n_valid);
      PROBE_REQUIRE(c.batches == 1, "split image: one batch");
      if ((rc = check_vec(c, c.bias, c.n_valid, "bias"))) return rc;
      return check_split_img(c, c.m, c.n_valid);
    case SKY_PROBE_EPI_F32_STATS: {
      PROBE_REQUIRE(c.n_valid % 8 == 0 && c.batches == 1 && c.ldo % 4 == 0 && c.ldo >= c.n_valid, "fp32 + image + statistics layout");
      const long long need = (c.m - 1) * c.ldo + c.n_valid;
      PROBE_REQUIRE(!c.out || (aligned16(c.out) && need * 4 <= c.out_bytes), "fp32 output too small");
      PROBE_REQUIRE(!c.add || (aligned16(c.add) && need * 4 <= c.add_bytes), "addend too small");
      PROBE_REQUIRE((c.asc == nullptr) == (c.ash == nullptr), "asc / ash");
      if ((rc = check_vec(c, c.bias, c.n_valid, "bias"))) return rc;
      if (c.asc && ((rc = check_vec(c, c.asc, c.n_valid, "asc")) || (rc = check_vec(c, c.ash, c.n_valid, "ash")))) return rc;
      if ((rc = check_sums(c))) return rc;
      return check_split_img(c, c.m, c.n_valid);
    }
    case SKY_PROBE_EPI_GELU_STATS: {
      PROBE_REQUIRE(c.n_valid % 8 == 0 && c.rows_per_batch >= 0 && (c.batches == 1 || c.rows_per_batch >= c.m), "GELU + statistics layout");
      const long long pixels = (long long)(c.batches - 1) * c.rows_per_batch + c.m;
      PROBE_REQUIRE(!c.add || (aligned16(c.add) && c.ldo % 4 == 0 && c.ldo >= c.n_valid && ((pixels - 1) * c.ldo + c.n_valid) * 4 <= c.add_bytes),
                    "addend too small");
      if (c.bias && (rc = check_vec(c, c.bias, c.n_valid, "bias"))) return rc;
      PROBE_REQUIRE(c.sums, "statistics pointer");
      if ((rc = check_sums(c))) return rc;
      return check_split_img(c, pixels, c.n_valid);
    }
    case SKY_PROBE_EPI_REMAP: {
      PROBE_REQUIRE(c.n_valid % 8 == 0 && c.bdiv >= 1 && c.kdiv >= 1 && c.kmul >= 0 && c.rb >= 0 && c.img_batch_bytes >= 0 &&
                        c.img_batch_bytes % 16 == 0 && (c.kdiv >= c.n_valid || c.kdiv % 8 == 0),
                    "remap parameters");
      long long db, drow, k;
      if (c.same) { db = c.batches - 1; drow = c.m - 1; k = c.n_valid - 1; }
      else {
        db = (c.m - 1) / c.bdiv;
        drow = (long long)(c.batches - 1) * c.rb + (c.n_valid - 1) / c.kdiv;
        k = (long long)((c.m < c.bdiv ? c.m : c.bdiv) - 1) * c.kmul + ((c.n_valid < c.kdiv ? c.n_valid : c.kdiv) - 1);
      }
      PROBE_REQUIRE(c.hi && c.lo && aligned16(c.hi) && aligned16(c.lo) && c.img_nkb >= 1 && k < c.img_nkb * 64LL, "remap destination");
      PROBE_REQUIRE(db * c.img_batch_bytes + (drow / 128 + 1) * c.img_nkb * TILE <= c.img_bytes, "remap destination too small");
      if (c.csc) {
        if ((rc = check_vec(c, c.csc, c.n_valid, "csc")) || (rc = check_vec(c, c.csh, c.n_valid, "csh"))) return rc;
        PROBE_REQUIRE(c.t1 && c.t1_floats >= c.m, "t1 shorter than M");
      }
      return 0;
    }
    case SKY_PROBE_EPI_LN:
    case SKY_PROBE_EPI_LN_IMG:
    case SKY_PROBE_EPI_LN_IMG_FRAG: {
      PROBE_REQUIRE(c.n_valid == c.n && c.batches == 1 && c.n <= 512, "LayerNorm: whole rows, one batch, N <= 512");
      PROBE_REQUIRE(c.kernel == SKY_PROBE_PAIR || c.n == c.block_n, "LayerNorm: one n-tile spans the row (N=%d, BN=%d)", c.n, c.block_n);
      if ((rc = check_vec(c, c.bias, c.n, "bias")) || (rc = check_vec(c, c.gamma, c.n, "gamma")) || (rc = check_vec(c, c.beta, c.n, "beta")))
        return rc;
      PROBE_REQUIRE(c.hi && aligned16(c.hi), "LayerNorm: fp16 image");
      if (c.epi == SKY_PROBE_EPI_LN)
        PROBE_REQUIRE(c.out && aligned16(c.out) && c.ldo % 4 == 0 && c.ldo >= c.n && ((c.m - 1) * c.ldo + c.n) * 4 <= c.out_bytes,
                      "LayerNorm: fp32 rows too small");
      return check_img(c, c.m, c.n);
    }
    case SKY_PROBE_EPI_F16_GELU_IMG:
    case SKY_PROBE_EPI_F16_GELU_IMG_FRAG:
    case SKY_PROBE_EPI_F16_ROWS: {
      PROBE_REQUIRE(c.n_valid == c.n && c.batches == 1, "fp16 output: every column, one batch");
      if ((rc = check_vec(c, c.bias, c.n, "bias"))) return rc;
      if (c.epi != SKY_PROBE_EPI_F16_ROWS) {
        PROBE_REQUIRE(c.hi && aligned16(c.hi), "fp16 image");
        return check_img(c, c.m, c.n);
      }
      PROBE_REQUIRE(c.out && aligned16(c.out) && c.ldo % 8 == 0 && c.ldo >= c.n && ((c.m - 1) * c.ldo + c.n) * 2 <= c.out_bytes,
                    "fp16 rows too small");
      return 0;
    }
    case SKY_PROBE_EPI_GC_SILU0:
    case SKY_PROBE_EPI_GC_SILU2: {
      PROBE_REQUIRE(c.n == GC_L && c.n_valid == c.n && c.batches == 1 && c.img_nkb == GC_NKB, "SiLU image: %d columns, %d k-blocks", GC_L, GC_NKB);
      PROBE_REQUIRE(c.hi && aligned16(c.hi), "SiLU image");
      if ((rc = check_vec(c, c.bias, c.n, "bias")) || (rc = check_img(c, c.m, c.n))) return rc;
      if (c.epi == SKY_PROBE_EPI_GC_SILU2 && (rc = check_gathers(c))) return rc;
      return 0;
    }
    case SKY_PROBE_EPI_GC_OUT: {
      PROBE_REQUIRE(c.batches == 1 && c.nprog >= 1 && c.nprog <= c.n && c.plane >= c.m, "output head: nprog %d, plane %lld", c.nprog,
                    (long long)c.plane);
      const long long need = ((long long)(c.nprog - 1) * c.plane + c.m) * 4;
      PROBE_REQUIRE(c.out && c.xin && need <= c.out_bytes && need <= c.xin_bytes, "output head planes too small");
      if ((rc = check_vec(c, c.bias, c.nprog, "bias")) || (rc = check_vec(c, c.dstd, c.nprog, "dstd"))) return rc;
      return 0;
    }
    case SKY_PROBE_EPI_GC_LN0:
    case SKY_PROBE_EPI_GC_LN1:
    case SKY_PROBE_EPI_GC_LN2: {
      PROBE_REQUIRE(c.kernel == SKY_PROBE_PAIR && c.n == GC_L && c.n_valid == c.n, "GraphCast LayerNorm: CTA pairs over %d columns", GC_L);
      if ((rc = check_vec(c, c.bias, c.n, "bias")) || (rc = check_vec(c, c.gamma, c.n, "gamma")) || (rc = check_vec(c, c.beta, c.n, "beta")))
        return rc;
      const long long rows_bytes = c.m * GC_L * 4, img_need = cdiv(c.m, G2_BLOCK_M) * GC_NKB * TILE;
      PROBE_REQUIRE(!c.out || (aligned16(c.out) && rows_bytes <= c.out_bytes), "fp32 rows too small");
      PROBE_REQUIRE((!c.hi || (aligned16(c.hi) && img_need <= c.img_bytes)) && (!c.yimg || (aligned16(c.yimg) && img_need <= c.img_bytes)),
                    "images too small");
      if (c.epi == SKY_PROBE_EPI_GC_LN1) PROBE_REQUIRE(c.xin && aligned16(c.xin) && rows_bytes <= c.xin_bytes, "fp32 residual rows");
      if (c.epi == SKY_PROBE_EPI_GC_LN2) PROBE_REQUIRE(c.xin_img && aligned16(c.xin_img) && img_need <= c.xin_bytes, "residual image");
      return 0;
    }
    case SKY_PROBE_EPI_QKV_WIN: {
      const char* ge = probe_geo_error(c.geo, c.pairs);
      PROBE_REQUIRE(!ge, "QKV window image: Geo: %s", ge ? ge : "");
      PROBE_REQUIRE(c.n == 3 * c.geo.C && c.n_valid == c.n && c.batches == 1, "QKV window image: N=%d is not 3C=%d, or n_valid / batches",
                    c.n, 3 * c.geo.C);
      PROBE_REQUIRE(c.roll == 0 || c.roll == 1, "QKV window image: roll %d", c.roll);
      // an n-tile of the fragment epilogue is three head pairs of one part
      PROBE_REQUIRE(c.geo.C % 192 == 0, "QKV window image: C=%d is not a multiple of 192", c.geo.C);
      PROBE_REQUIRE(c.m % c.geo.T == 0, "QKV window image: M=%lld is not members x T=%d", (long long)c.m, c.geo.T);
      // the epilogue's 32-bit row arithmetic: members x tokens and members x windows x pairs x 144 rows below 2^31
      const long long tiles = c.m / c.geo.T * c.geo.nWin * c.pairs;
      PROBE_REQUIRE(c.m < (1LL << 31) && tiles * WIN_TOK < (1LL << 31), "QKV window image: %lld tiles overflow 32-bit rows", tiles);
      PROBE_REQUIRE(c.part_stride >= tiles * AT_TILE_B && c.part_stride % 16 == 0, "QKV window image: part stride %lld (%lld tiles)",
                    (long long)c.part_stride, tiles);
      PROBE_REQUIRE(c.hi && aligned16(c.hi) && 2 * c.part_stride + tiles * AT_TILE_B <= c.img_bytes, "QKV window image too small");
      return check_vec(c, c.bias, c.n, "bias");
    }
    default:
      PROBE_REQUIRE(false, "unknown epilogue %d", c.epi);
  }
  return 0;
}

// ---- dispatch ----
// the first device call of the probe: everything before it is host-side validation
template <int BN, bool kPair, class Sched, class Epi>
int run(const Case& c, const Sched& sc, const Epi& e, cudaStream_t st) {
  int sms = c.grid_sms;
  if (sms == 0) {
    int dev = 0;
    SKY_CUDA_OK(cudaGetDevice(&dev));
    SKY_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  return launch_gemm2<BN, kPair>(sc, e, c.m, c.n, c.batches, sms, st);
}

template <class Epi>
Epi make_epi(const Case& c);
template <> EpiF32Batched<false> make_epi(const Case& c) { return {(float*)c.out, c.ldo, c.out_batch_stride, c.bias, c.n_valid, c.add}; }
template <> EpiF32Batched<true> make_epi(const Case& c) { return {(float*)c.out, c.ldo, c.out_batch_stride, c.bias, c.n_valid, c.add}; }
template <> EpiSplitImg<false> make_epi(const Case& c) { return {(uint8_t*)c.hi, (uint8_t*)c.lo, c.img_nkb, c.bias, c.n_valid}; }
template <> EpiSplitImg<true> make_epi(const Case& c) { return {(uint8_t*)c.hi, (uint8_t*)c.lo, c.img_nkb, c.bias, c.n_valid}; }
template <> EpiF32ImgStats make_epi(const Case& c) {
  return {(float*)c.out, c.ldo, (uint8_t*)c.hi, (uint8_t*)c.lo, c.img_nkb, c.bias, c.add, c.asc, c.ash, c.sums, c.n_valid};
}
template <> EpiGeluStatsImg make_epi(const Case& c) {
  return {(uint8_t*)c.hi, (uint8_t*)c.lo, c.img_nkb, c.bias, c.add, c.ldo, c.rows_per_batch, c.sums, c.n_valid};
}
template <> EpiSplitRemap make_epi(const Case& c) {
  return {(uint8_t*)c.hi, (uint8_t*)c.lo, c.img_batch_bytes, c.img_nkb, c.bdiv, c.kmul, c.kdiv, c.rb, c.n_valid, c.same, c.csc, c.csh, c.t1};
}
// The LayerNorm epilogue as Pangu runs it (make_ln): in place on fp32 rows `out` and their image `hi`, or on the image
// `hi` alone; and as GraphCast runs it (make_gcln): the residual from xin or xin_img, any of out, hi and yimg written, rows
// of 512 and 8 k-blocks.  Epi2F32Img<true, 1 / 2> serves both, so these are not make_epi specialisations.
template <int kRes>
Epi2F32Img<true, kRes> make_ln(const Case& c) {
  return {kRes == 1 ? c.out : c.hi, kRes == 1 ? (float*)c.out : nullptr, c.ldo, (uint8_t*)c.hi, c.img_nkb, nullptr, c.bias, c.gamma, c.beta, c.eps};
}
template <int kRes>
Epi2F32Img<true, kRes> make_gcln(const Case& c) {
  const void* res = kRes == 1 ? static_cast<const void*>(c.xin) : c.xin_img;
  return {res, (float*)c.out, GC_L, (uint8_t*)c.hi, GC_NKB, (uint8_t*)c.yimg, c.bias, c.gamma, c.beta, c.eps};
}

template <> Epi2F16<true, true> make_epi(const Case& c) { return {(__half*)c.hi, 0, c.img_nkb, c.bias}; }
template <> Epi2F16<false, false> make_epi(const Case& c) { return {(__half*)c.out, c.ldo, 0, c.bias}; }
template <> FragEpi<Epi2F16<true, true>> make_epi(const Case& c) { return {make_epi<Epi2F16<true, true>>(c)}; }
template <int kG>
EpiGcSiluImg<kG> make_silu(const Case& c) {
  EpiGcSiluImg<kG> e{};
  e.out = (uint8_t*)c.hi; e.bias = c.bias;
  e.ta = (const __half*)c.ta; e.lda = c.lda; e.ia = c.ia; e.tb = (const __half*)c.tb; e.ldb = c.ldb; e.ib = c.ib;
  return e;
}
template <> EpiGcSiluImg<0> make_epi(const Case& c) { return make_silu<0>(c); }
template <> EpiGcSiluImg<2> make_epi(const Case& c) { return make_silu<2>(c); }
template <> EpiGcOut make_epi(const Case& c) {
  EpiGcOut e{};
  e.xout = (float*)c.out; e.xin = c.xin; e.bias = c.bias; e.dstd = c.dstd; e.plane = c.plane; e.nprog = c.nprog;
  return e;
}
template <> FragEpi<EpiQkvWin> make_epi(const Case& c) {
  return {EpiQkvWin{(uint8_t*)c.hi, c.part_stride, c.bias, probe_geo(c.geo), c.roll, c.geo.C, c.pairs}};
}

// ---- the fused MLP (SKY_PROBE_MLP) ----
int check_mlp(const Case& c) {
  const int C = c.n;
  PROBE_REQUIRE((C == 192 || C == 384) && c.m >= 1 && c.grid_sms >= 0, "fused MLP: N=%d (must be 192 or 384), M=%lld, grid_sms %d", C,
                (long long)c.m, c.grid_sms);
  PROBE_REQUIRE(C == 192 || c.grid_sms != 1, "fused MLP: grid_sms 1 (CTA pairs at N=384)");
  PROBE_REQUIRE(c.img_nkb == C / 64 && c.hi && aligned16(c.hi) && cdiv(c.m, G2_BLOCK_M) * (C / 64) * TILE <= c.img_bytes,
                "fused MLP: stream image too small or not %d k-blocks", C / 64);
  const long long wbytes = 4LL * C * C * 2;
  PROBE_REQUIRE(c.w && aligned16(c.w) && c.w_bytes >= wbytes && c.b_hi && aligned16(c.b_hi) && c.b_bytes >= wbytes,
                "fused MLP: weight images of %lld bytes", wbytes);
  PROBE_REQUIRE(c.add && aligned16(c.add) && c.add_bytes >= 4LL * C * 4, "fused MLP: fc1 bias of %d floats", 4 * C);
  int rc;
  if ((rc = check_vec(c, c.bias, C, "bias")) || (rc = check_vec(c, c.gamma, C, "gamma")) || (rc = check_vec(c, c.beta, C, "beta")))
    return rc;
  return 0;
}
int run_mlp(const Case& c, cudaStream_t st) {
  int sms = c.grid_sms;
  if (sms == 0) {
    int dev = 0;
    SKY_CUDA_OK(cudaGetDevice(&dev));
    SKY_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const MlpArgs a{(uint8_t*)c.hi, (const uint8_t*)c.w, (const uint8_t*)c.b_hi, c.add, {make_ln<2>(c)}, c.m};
  return c.n == 192 ? launch_mlp_fused<3>(a, sms, st) : launch_mlp_fused_pair(a, sms, st);
}

template <int... BNs> struct BnList {};

// launch epilogue e with the case's BLOCK_N if it is in the list, else refuse
template <bool kPair, class Sched, class Epi, int... BNs>
int launch_bn(const Case& c, const Sched& sc, const Epi& e, cudaStream_t st, BnList<BNs...>) {
  int rc = -1;
  ((c.block_n == BNs ? (rc = run<BNs, kPair>(c, sc, e, st), 0) : 0), ...);
  if (rc == -1) {
    set_error("gemm probe: BLOCK_N %d is not instantiated for kernel %d / epilogue %d", c.block_n, c.kernel, c.epi);
    return SKY_ERR_ARG;
  }
  return rc;
}
template <bool kPair, class Epi, class Sched, class Bns>
int by_bn(const Case& c, const Sched& sc, cudaStream_t st, Bns bns) {
  return launch_bn<kPair>(c, sc, make_epi<Epi>(c), st, bns);
}

// The (schedule, epilogue, BLOCK_N) lists mirror what the engines instantiate:
//   SFNO SfnoEngine::gemm_op: SchedW / SchedW<true> x its epilogues x {16, 32, 64, 80, 192, 240, 256};
//   SFNO SfnoEngine::gemm_tb: SchedTB x {EpiSplitRemap, EpiF32Batched<false>, EpiGeluStatsImg} x {64, 128, 192, 256};
//   Pangu: SchedW x Epi2F32Img<true, 1 / 2> at 192, and the pair kernel at 192; fc1's Epi2F16<true, true> at 192; the
//   fragment path of the QKV projection (FragEpi<EpiQkvWin>, which has no staged form), of the projection / fc2
//   (FragEpi<Epi2F32Img<true, 2>>, single CTA and pair) and of fc1 (FragEpi<Epi2F16<true, true>>) at 192.  The engine
//   launches the staged Epi2F32Img<true, 2> only at 256 (GraphCast) and Epi2F16<true, true> not at all; the probe keeps
//   them at 192 as the reference of the fragment path;
//   GraphCast: EpiGcSiluImg<0 / 2> and the node tables' Epi2F16<false, false> at 256, EpiGcOut at 128, and the pair kernel
//   with Epi2F32Img<true, 0 / 1 / 2> at 256 (GraphCast never gathers exactly one table: EpiGcSiluImg<1> is not
//   instantiated).
using BnSfno = BnList<16, 32, 64, 80, 192, 240, 256>;
using BnSfnoMain = BnList<64, 192>;
using BnTb = BnList<64, 128, 192, 256>;
using BnPair = BnList<192>;

int dispatch(const Case& c, cudaStream_t st) {
  if (c.kernel == SKY_PROBE_TB) {
    const SchedTB sc{(const uint8_t*)c.t, c.t_batch_stride,
                     BData{(const uint8_t*)c.b_hi, (const uint8_t*)c.b_lo, c.b_nkb_img, c.b_rows_per_batch, c.b_batch_bytes}, c.num_kb};
    switch (c.epi) {
      case SKY_PROBE_EPI_REMAP: return by_bn<false, EpiSplitRemap>(c, sc, st, BnTb{});
      case SKY_PROBE_EPI_F32: return by_bn<false, EpiF32Batched<false>>(c, sc, st, BnTb{});
      case SKY_PROBE_EPI_GELU_STATS: return by_bn<false, EpiGeluStatsImg>(c, sc, st, BnTb{});
      default: break;
    }
  } else {
    AOperand a;
    for (int s = 0; s < c.nseg; ++s) a.add((const uint8_t*)c.a[s], c.a_nkb[s], c.a_batch_stride[s]);
    if (c.kernel == SKY_PROBE_W_TRI) {
      const SchedW<true> sc{a, (const uint8_t*)c.w, c.num_kb, c.w_batch_stride, c.w_rep};
      if (c.epi == SKY_PROBE_EPI_REMAP) return by_bn<false, EpiSplitRemap>(c, sc, st, BnSfnoMain{});
    } else {
      const SchedW<false> sc{a, (const uint8_t*)c.w, c.num_kb, c.w_batch_stride, c.w_rep};
      if (c.kernel == SKY_PROBE_PAIR) {
        switch (c.epi) {
          case SKY_PROBE_EPI_LN: return launch_bn<true>(c, sc, make_ln<1>(c), st, BnPair{});
          case SKY_PROBE_EPI_LN_IMG: return launch_bn<true>(c, sc, make_ln<2>(c), st, BnPair{});
          case SKY_PROBE_EPI_LN_IMG_FRAG: return launch_bn<true>(c, sc, FragEpi<Epi2F32Img<true, 2>>{make_ln<2>(c)}, st, BnPair{});
          case SKY_PROBE_EPI_GC_LN0: return launch_bn<true>(c, sc, make_gcln<0>(c), st, BnList<256>{});
          case SKY_PROBE_EPI_GC_LN1: return launch_bn<true>(c, sc, make_gcln<1>(c), st, BnList<256>{});
          case SKY_PROBE_EPI_GC_LN2: return launch_bn<true>(c, sc, make_gcln<2>(c), st, BnList<256>{});
          default: break;
        }
      } else if (c.kernel == SKY_PROBE_W) {
        switch (c.epi) {
          case SKY_PROBE_EPI_F32: return by_bn<false, EpiF32Batched<false>>(c, sc, st, BnSfno{});
          case SKY_PROBE_EPI_F32_ACC: return by_bn<false, EpiF32Batched<true>>(c, sc, st, BnSfno{});
          case SKY_PROBE_EPI_SPLIT: return by_bn<false, EpiSplitImg<false>>(c, sc, st, BnSfnoMain{});
          case SKY_PROBE_EPI_SPLIT_GELU: return by_bn<false, EpiSplitImg<true>>(c, sc, st, BnSfnoMain{});
          case SKY_PROBE_EPI_F32_STATS: return by_bn<false, EpiF32ImgStats>(c, sc, st, BnSfnoMain{});
          case SKY_PROBE_EPI_GELU_STATS: return by_bn<false, EpiGeluStatsImg>(c, sc, st, BnSfnoMain{});
          case SKY_PROBE_EPI_LN: return launch_bn<false>(c, sc, make_ln<1>(c), st, BnList<192>{});
          case SKY_PROBE_EPI_LN_IMG: return launch_bn<false>(c, sc, make_ln<2>(c), st, BnList<192>{});
          case SKY_PROBE_EPI_F16_GELU_IMG: return by_bn<false, Epi2F16<true, true>>(c, sc, st, BnList<192>{});
          case SKY_PROBE_EPI_LN_IMG_FRAG: return launch_bn<false>(c, sc, FragEpi<Epi2F32Img<true, 2>>{make_ln<2>(c)}, st, BnList<192>{});
          case SKY_PROBE_EPI_F16_GELU_IMG_FRAG: return by_bn<false, FragEpi<Epi2F16<true, true>>>(c, sc, st, BnList<192>{});
          case SKY_PROBE_EPI_F16_ROWS: return by_bn<false, Epi2F16<false, false>>(c, sc, st, BnList<256>{});
          case SKY_PROBE_EPI_GC_SILU0: return by_bn<false, EpiGcSiluImg<0>>(c, sc, st, BnList<256>{});
          case SKY_PROBE_EPI_GC_SILU2: return by_bn<false, EpiGcSiluImg<2>>(c, sc, st, BnList<256>{});
          case SKY_PROBE_EPI_GC_OUT: return by_bn<false, EpiGcOut>(c, sc, st, BnList<128>{});
          case SKY_PROBE_EPI_QKV_WIN: return by_bn<false, FragEpi<EpiQkvWin>>(c, sc, st, BnList<192>{});
          default: break;
        }
      }
    }
  }
  set_error("gemm probe: kernel %d with epilogue %d is not instantiated", c.kernel, c.epi);
  return SKY_ERR_ARG;
}

}  // namespace
}  // namespace sky

extern "C" SKY_API int sky_probe_gemm(const sky_probe_case_t* c, void* stream) {
  using namespace sky;
  if (!c) { set_error("gemm probe: null case"); return SKY_ERR_ARG; }
  if (c->kernel < SKY_PROBE_W || c->kernel > SKY_PROBE_MLP) { set_error("gemm probe: unknown kernel %d", c->kernel); return SKY_ERR_ARG; }
  int rc;
  if (c->kernel == SKY_PROBE_MLP) return (rc = check_mlp(*c)) ? rc : run_mlp(*c, (cudaStream_t)stream);
  if ((rc = check_operands(*c)) || (rc = check_epilogue(*c))) return rc;
  return dispatch(*c, (cudaStream_t)stream);
}
