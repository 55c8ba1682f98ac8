// Kernel-level probe of Pangu's windowing kernels, for tests only: part of libskyrim_b200_probe.so.
//
// sky_probe_pangu makes ONE launch of a kernel that is not a k_gemm2 epilogue, from raw device pointers, so that
// tests/test_pangu_kernels_gpu.py can compare it element by element against oracle/pangu_kernels_ref.py:
//   FILL_PAD    k_qkv_fill_pad: the q / k / v rows of latitude-padding tokens in the window image = the QKV bias
//   ATTENTION   k_window_attention_tc: window image + compact fp16 bias tables -> (tokens, C) operand image; one CTA per
//               SM, or a chosen number of CTAs through sky_probe_pangu_grid
//   PACK_BIAS   k_pack_bias_table: fp32 (3312, type, head) -> fp16 (type, head, 3312) x log2 e
// (The QKV projection's epilogue EpiQkvWin is reached through sky_probe_gemm.)  The kernels are launched through the
// engine's own host launchers (attention_tc.cuh, defined in pangu_engine.o), so each has one definition.
//
// A case is validated on the host before anything touches the device; an inconsistent one is refused with an error
// (sky_last_error) instead.
#include <cstdint>

#include "gemm2.cuh"
#include "attention_tc.cuh"
#include "probe_geo.cuh"

extern "C" {

enum { SKY_PROBE_PG_FILL_PAD = 0, SKY_PROBE_PG_ATTENTION = 1, SKY_PROBE_PG_PACK_BIAS = 2 };

// Every pointer is a device pointer; every *_bytes / *_floats field is the size of the allocation behind it.
typedef struct {
  int32_t op;
  sky_probe_geo_t geo;
  int32_t roll, B, pairs;
  int32_t n_type;            // bias tables: window types (nWz x nWh), heads = geo.heads
  int32_t att_nkb;           // ATTENTION: 64-column blocks of the output image (>= pairs)
  int64_t part_stride;       // bytes between the q, k and v parts of the window image
  void* qkv; int64_t qkv_bytes;            // window image: written by FILL_PAD, read by ATTENTION
  const float* src; int64_t src_floats;    // FILL_PAD: QKV bias (3C); PACK_BIAS: fp32 table (3312, n_type, heads)
  const void* tab; int64_t tab_bytes;      // ATTENTION: fp16 tables (n_type, heads, 3312), pre-scaled by log2 e
  void* out; int64_t out_bytes;            // ATTENTION: fp16 tile image (B T, C); PACK_BIAS: fp16 tables
  float sl2, mask_l2;        // ATTENTION: head_dim^-0.5 log2 e and mask value x log2 e
} sky_probe_pangu_t;

SKY_API int sky_probe_pangu_size(void) { return (int)sizeof(sky_probe_pangu_t); }
SKY_API int sky_probe_pangu(const sky_probe_pangu_t* c, void* stream);
// sky_probe_pangu with the persistent attention kernel's grid set to grid_ctas CTAs (at most one per item); 0 = one per SM
SKY_API int sky_probe_pangu_grid(const sky_probe_pangu_t* c, int32_t grid_ctas, void* stream);

}  // extern "C"

namespace sky {
namespace {

// The compact table index the attention kernel forms, (query part) + (key part), spans exactly [0, AT_TABLE): the
// largest is (zi, hi, wi) = (1, 5, 11) against (zj, hj, wj) = (1, 5, 0), the smallest wi = 0 against wj = 11.  So no
// case can read a bias entry outside the (type, head) table it expands.
static_assert((WZ - 1) * (1 + WZ) * ((2 * WW - 1) * WH * WH) + (WH - 1) * (1 + WH) * (2 * WW - 1) + 2 * (WW - 1) == AT_TABLE - 1,
              "bias table index range");

#define PG_REQUIRE(cond, ...)                    \
  do {                                           \
    if (!(cond)) {                               \
      set_error("pangu probe: " __VA_ARGS__);    \
      return SKY_ERR_ARG;                        \
    }                                            \
  } while (0)

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

// the window image: 3 parts of members x windows x pairs tiles of 144 rows x 128 B
int check_window_image(const sky_probe_pangu_t& c) {
  const long long tiles = (long long)c.B * c.geo.nWin * c.pairs;
  PG_REQUIRE(tiles * WIN_TOK < (1LL << 31), "%lld window tiles overflow 32-bit rows", tiles);
  PG_REQUIRE(c.part_stride >= tiles * AT_TILE_B && c.part_stride % 16 == 0, "part stride %lld (%lld tiles)", (long long)c.part_stride, tiles);
  PG_REQUIRE(c.qkv && aligned16(c.qkv) && 2 * c.part_stride + tiles * AT_TILE_B <= c.qkv_bytes, "window image too small");
  return 0;
}

int check(const sky_probe_pangu_t& c) {
  PG_REQUIRE(c.op >= SKY_PROBE_PG_FILL_PAD && c.op <= SKY_PROBE_PG_PACK_BIAS, "unknown op %d", c.op);
  const char* ge = probe_geo_error(c.geo, c.pairs);
  PG_REQUIRE(!ge, "Geo: %s", ge ? ge : "");
  PG_REQUIRE(c.B >= 1 && (long long)c.B * c.geo.T < (1LL << 31), "members %d (T %d)", c.B, c.geo.T);
  PG_REQUIRE(c.roll == 0 || c.roll == 1, "roll %d", c.roll);
  const long long n_tab = (long long)AT_TABLE * c.n_type * c.geo.heads;
  int rc;
  switch (c.op) {
    case SKY_PROBE_PG_FILL_PAD:
      PG_REQUIRE(c.geo.Hp > c.geo.H, "no latitude padding (H=%d = Hp)", c.geo.H);
      if ((rc = check_window_image(c))) return rc;
      PG_REQUIRE(c.src && c.src_floats >= 3LL * c.geo.C, "QKV bias shorter than 3C");
      return 0;
    case SKY_PROBE_PG_ATTENTION: {
      if ((rc = check_window_image(c))) return rc;
      PG_REQUIRE(c.n_type == c.geo.nWz * c.geo.nWh, "%d bias window types, the grid has %d", c.n_type, c.geo.nWz * c.geo.nWh);
      PG_REQUIRE(c.tab && aligned16(c.tab) && n_tab * 2 <= c.tab_bytes, "bias tables too small");
      PG_REQUIRE(c.att_nkb >= c.pairs, "output image: %d k-blocks for %d head pairs", c.att_nkb, c.pairs);
      const long long rows = (long long)c.B * c.geo.T;
      PG_REQUIRE(c.out && aligned16(c.out) && (rows + 127) / 128 * c.att_nkb * (long long)G2_A_BYTES <= c.out_bytes, "output image too small");
      PG_REQUIRE(c.sl2 == c.sl2 && c.mask_l2 == c.mask_l2, "NaN scale or mask");
      return 0;
    }
    case SKY_PROBE_PG_PACK_BIAS:
      PG_REQUIRE(c.n_type == c.geo.nWz * c.geo.nWh, "%d bias window types, the grid has %d", c.n_type, c.geo.nWz * c.geo.nWh);
      PG_REQUIRE(c.src && c.src_floats >= n_tab, "fp32 table shorter than 3312 x types x heads");
      PG_REQUIRE(c.out && n_tab * 2 <= c.out_bytes, "fp16 tables too small");
      return 0;
  }
  return 0;
}

int dispatch(const sky_probe_pangu_t& c, int grid_ctas, cudaStream_t st) {
  const Geo g = probe_geo(c.geo);
  switch (c.op) {
    case SKY_PROBE_PG_FILL_PAD:
      return launch_qkv_fill_pad((uint8_t*)c.qkv, c.part_stride, c.src, g, c.roll, c.B, c.pairs, st);
    case SKY_PROBE_PG_ATTENTION: {
      const AttnArgs a{(const uint8_t*)c.qkv, c.part_stride, (uint8_t*)c.out, c.att_nkb, (const __half*)c.tab, g, c.roll, c.B, c.pairs,
                       c.sl2, c.mask_l2, (long long)c.B * g.nWin * c.pairs};
      return launch_window_attention_tc(a, grid_ctas, st);
    }
    case SKY_PROBE_PG_PACK_BIAS:
      return launch_pack_bias_table(c.src, (__half*)c.out, c.n_type, g.heads, st);
  }
  return SKY_ERR_ARG;
}

}  // namespace
}  // namespace sky

extern "C" SKY_API int sky_probe_pangu_grid(const sky_probe_pangu_t* c, int32_t grid_ctas, void* stream) {
  using namespace sky;
  if (!c) { set_error("pangu probe: null case"); return SKY_ERR_ARG; }
  if (grid_ctas < 0) { set_error("pangu probe: grid of %d CTAs", grid_ctas); return SKY_ERR_ARG; }
  if (int rc = check(*c)) return rc;
  return dispatch(*c, grid_ctas, (cudaStream_t)stream);
}

extern "C" SKY_API int sky_probe_pangu(const sky_probe_pangu_t* c, void* stream) { return sky_probe_pangu_grid(c, 0, stream); }
