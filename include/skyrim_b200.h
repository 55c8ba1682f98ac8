/* skyrim_b200 — C-ABI of the H100 (sm_90a) step operators behind the Skyrim rollout path.
 *
 * The reference has no FFI of its own: its seam is the Python earth2mip ``TimeLoop``
 * protocol consumed at
 *   /root/reference/skyrim/core/models/utils.py:34-40   (for k,(time,output,_) in model(time,x))
 *   /root/reference/skyrim/core/models/pangu.py:45-46   (pangu.load(registry.get_model(...)))
 *   /root/reference/skyrim/core/models/fourcastnet_v2.py:36-37
 * Each entry point below replaces what one of those call sites reaches inside the
 * ONNXRuntime / earth2mip back-ends.  Plain pointers and sizes only; no Python or torch
 * types cross this boundary.  Device pointers are raw CUDA device addresses (the Python
 * host passes ``tensor.data_ptr()``), ``stream`` is a ``cudaStream_t`` cast to void*.
 *
 * Conventions: every function returns 0 on success, <0 on error (never exits);
 * sky_last_error() returns a thread-local message.  A handle is bound to one device and is
 * not thread-safe; distinct handles on distinct devices may be driven concurrently.
 * The caller owns state / workspace buffers; the engine owns its device weights.
 */
#ifndef SKYRIM_B200_H
#define SKYRIM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SKY_ABI_VERSION 1

enum { SKY_MODEL_PANGU6 = 1, SKY_MODEL_SFNO73 = 2, SKY_MODEL_GRAPHCAST = 3 };
enum { SKY_OK = 0, SKY_ERR_ARG = -1, SKY_ERR_CUDA = -2, SKY_ERR_STATE = -3, SKY_ERR_NOMEM = -4 };

/* Pangu-Weather 6-h operator shape (patch (2,4,4) and window (2,6,12) are fixed).
 * Replaces the shape information baked into pangu_weather_6.onnx (pangu.py:46). */
typedef struct {
  int32_t nlat, nlon;      /* 721, 1440 */
  int32_t n_levels;        /* 13 */
  int32_t dim;             /* 192 */
  int32_t depths[4];       /* 2,6,6,2 */
  int32_t heads[4];        /* 6,12,12,6 */
  float ln_eps;            /* 1e-5 */
  float mask_value;        /* -100 */
} sky_pangu_config_t;

/* SFNO (FourCastNet-v2-small) operator shape; replaces the hyper-parameters read from the
 * fcnv2_sm checkpoint (fourcastnet_v2.py:37). */
typedef struct {
  int32_t nlat, nlon;      /* 721, 1440 */
  int32_t n_channels;      /* 73 */
  int32_t embed;           /* 384 */
  int32_t layers;          /* 8 */
  int32_t scale_factor;    /* 3 */
  int32_t mlp_ratio;       /* 2 */
  float eps;               /* instance-norm epsilon */
} sky_sfno_config_t;

/* GraphCast (operational 0.25 deg / 13 levels) operator shape; replaces what
 * graphcast.load_time_loop_operational reads from the checkpoint and builds as mesh tables
 * (/root/reference/skyrim/core/models/graphcast.py:51-54).  The graph itself (edge lists, edge / node features)
 * travels in the weight arena as entries named "graph.*" (skyrim_b200/icomesh.py); the counts below size them. */
typedef struct {
  int32_t nlat, nlon;      /* 721, 1440 */
  int32_t n_mesh;          /* 40962 multimesh nodes (icosahedron refined 6 times) */
  int32_t n_mesh_edges;    /* 327660 directed multimesh edges, sorted by receiver */
  int32_t n_g2m_edges;     /* grid2mesh edges, sorted by receiver (mesh node) */
  int32_t latent;          /* 512 */
  int32_t layers;          /* 16 processor layers */
  int32_t n_state;         /* 83 channels per time slice: 82 prognostic + toa radiation (graphcast.py:17-41) */
  int32_t n_prog;          /* 82 */
  int32_t n_static;        /* 2: geopotential at the surface, land-sea mask */
  int32_t dt_hours;        /* 6 */
  float ln_eps;            /* 1e-5 */
} sky_graphcast_config_t;
/* Arena entries of a GraphCast model (all fp32; index tables hold exact integers < 2^24):
 *   norm.mean, norm.std, norm.diff_std (n_state each), static.fields (n_static, nlat, nlon)
 *   <mlp>.w1 (512, fan_in), .b1 (512), .w2 (fan_out, 512), .b2 (fan_out), .ln.g / .ln.b (fan_out; not for dec.out) for <mlp> in
 *     enc.grid_embed (184), enc.mesh_embed (3), enc.g2m_edge_embed (4), enc.g2m_edge (1536), enc.g2m_mesh (1024), enc.g2m_grid (512),
 *     proc.edge_embed (4), proc<i>.edge (1536), proc<i>.node (1024) for i < layers, dec.m2g_edge_embed (4), dec.m2g_edge (1536),
 *     dec.m2g_grid (1024), dec.out (512 -> n_state)          [first-layer input order: edge | sender | receiver, node | aggregate]
 *   graph.mesh.senders / .receivers (n_mesh_edges, sorted by receiver), graph.mesh.ptr (n_mesh + 1), graph.mesh.edge_feat (n_mesh_edges, 4),
 *   graph.mesh.node_feat (n_mesh, 3), graph.g2m.senders / .receivers / .ptr / .edge_feat (same, grid -> mesh),
 *   graph.m2g.senders (3 * nlat * nlon, k-major: edge k of grid point g at k * n_grid + g), graph.m2g.edge_feat (3 * n_grid, 4),
 *   graph.grid.coslat (nlat), graph.grid.sinlon / .coslon (nlon)
 * (skyrim_b200/weights.py::graphcast_param_shapes, skyrim_b200/icomesh.py::graph_arena_entries build exactly this set). */

/* one named fp32 tensor inside a flat weight arena */
typedef struct {
  char name[96];
  uint64_t offset;         /* in floats from the arena start */
  uint64_t count;          /* number of floats */
} sky_param_desc_t;

typedef struct sky_model sky_model_t;

/* Everything but these entry points is built with hidden visibility: the product and the development build of the
 * library can then live in one process without their template statics / inline functions being merged by the
 * dynamic linker (round 2: a shared `configured` flag made the second library skip its shared-memory opt-in). */
#if defined(__GNUC__)
#define SKY_API __attribute__((visibility("default")))
#else
#define SKY_API
#endif

SKY_API int sky_abi_version(void);
SKY_API const char* sky_last_error(void);

/* model_kind: SKY_MODEL_*; cfg points at the matching sky_*_config_t. */
SKY_API int sky_model_create(sky_model_t** out, int model_kind, const void* cfg, size_t cfg_bytes, int device);

/* Load (copy + repack for the tensor cores) the fp32 weight arena.  `arena` is a host
 * pointer (arena_on_device = 0) or a device pointer on the model's device (= 1, e.g. the
 * buffer that received the one-time NCCL broadcast).  The caller keeps ownership.
 * Replaces ONNX initialiser loading / torch.load in the reference back-ends. */
SKY_API int sky_model_load_weights(sky_model_t* m, const float* arena, uint64_t n_floats,
                           const sky_param_desc_t* manifest, int32_t n_params, int32_t arena_on_device,
                           void* stream);

/* scratch bytes one step needs for `batch` members */
SKY_API size_t sky_model_workspace_bytes(const sky_model_t* m, int32_t batch);

/* One 6-h step for `batch` independent members: x_in, x_out are device fp32
 * (batch, C, nlat, nlon), may not alias.  Asynchronous and stream-ordered; no host sync.
 * Replaces one `next()` of the TimeLoop generator (utils.py:34). */
SKY_API int sky_model_step(sky_model_t* m, const float* x_in, float* x_out, int32_t batch, void* workspace,
                   size_t workspace_bytes, void* stream);

/* Valid time (unix seconds, UTC) of the LAST time slice of the state the next sky_model_step starts from.  Operators
 * with time-dependent forcings (GraphCast: toa radiation, year / day progress) keep this clock on the device and advance
 * it by one step per sky_model_step, so a rollout sets it once; the others ignore it.
 * Replaces the `time` argument of `stepper.initialize(x, time)` (graphcast.py:110). */
SKY_API int sky_model_set_clock(sky_model_t* m, double unix_seconds, void* stream);

/* Top-of-atmosphere incident solar radiation of the hour ending at `unix_seconds` [J m^-2] on the (nlat, nlon) grid
 * (lat 90 -> -90, lon 0 -> 360): the forcing channel the reference calls "tp06" (graphcast.py:16,40).  `out` is device
 * fp32 (nlat * nlon).  Used to fill that channel of an initial condition. */
SKY_API int sky_toa_radiation(float* out, int32_t nlat, int32_t nlon, double unix_seconds, void* stream);

/* Intermediate tensor taps for kernel-level parity tests: after a step, copy the named
 * internal buffer ("embed"/"tokens1"/"tokens2"...) of the LAST step into dst (device fp32). */
SKY_API int sky_model_debug_copy(sky_model_t* m, const char* what, float* dst, uint64_t max_floats, void* workspace,
                         int32_t batch, void* stream);

/* Switches of a handle (never read from the environment).  "fp32_stream" = 1 (Pangu) keeps the token stream as fp32 rows beside
 * its fp16 operand image instead of the default image-only stream: 1.1 ms per step slower, one rounding per residual add less
 * (DESIGN.md section 3).  Test taps: "stop_after" = n makes step() return after
 * stage n (Pangu: 0 embed, 1 layer0, 2 down, 3 layer1, 4 layer2, 5 up, 6 layer3; SFNO: 0 encoder, 1 + i block i;
 * 99 = run the whole step) so that sky_model_debug_copy can read the intermediate buffers.  GraphCast also takes
 * "stop_launch" = n: a member's step returns after its n-th unit in program order (the feature kernel, every hidden GEMM,
 * LayerNorm GEMM, per-node table and aggregation), because its workspace buffers are reused within a step; -1 = never.
 * Its debug_copy names "feat", "hid", "hid_m", "vg_img", "tg", "tm", "yimg", "ym_img", "em_img", "agg_img", "vm_img",
 * "vm0_img", "e_g2m_img", "e_m2g_img", "e_mesh_img" and "g2m_tr" copy the whole buffer as raw bytes (fp16 tile images,
 * fp16 row-major tables); max_floats must be its exact size. */
SKY_API int sky_model_debug_set(sky_model_t* m, const char* key, int64_t value);

/* x[m, c, :, :] += amp * sigma[c] * N(0,1), Philox4x32-10 keyed by (seed, member0 + m):
 * perturbed-IC ensemble members (new functionality; the reference's only perturbation
 * helper is the single-point edit at models/utils.py:70-92). */
SKY_API int sky_perturb_ic(float* x, const float* sigma_c, float amp, uint64_t seed, int32_t member0,
                   int32_t members, int32_t channels, int64_t plane, void* stream);

/* Spherically correlated perturbation: x[m, c, :, :] += amp * sigma[c] * f, f a Gaussian random field on the sphere with
 * unit pointwise variance, per field (global member g = member0 + m, channel c):
 *   a_l0 = s_l z0,  a_lm = s_l (z0 + i z1) / sqrt 2 (0 < m <= l <= lmax),  z0, z1 = fp64 Box-Muller of the first two
 *   words of Philox4x32-10 with key = seed and counter = (l | m << 16, 0x47524631 "GRF1", c, g),
 *   f = the inverse real SHT of a_lm on the equiangular (nlat, nlon) grid, torch-harmonics conventions
 *   (skyrim_b200/sht.py RealSHT.inverse).
 * A draw depends only on (seed, g, c, l, m): not on lmax, on the batch or on the rank layout.  Channels with
 * sigma[c] == 0 are left bit-identical.  All pointers are device memory on the device that owns x:
 *   spec_std   fp32 [lmax + 1], s_l (skyrim_b200.engine.grf_spectrum: s_0 = 0, sum_l s_l^2 (2l + 1) / 4 pi = 1);
 *   legendre   fp32 Pbar_l^m(cos theta_k) for m = 0..lmax, k < nlat, l = m..lmax, stored m-major, then k, then l
 *              (block m holds nlat * (lmax + 1 - m) values);
 *   workspace  at least sky_grf_workspace_bytes(members, channels, nlat, nlon, lmax) bytes (at most 512 MB whenever one
 *              field fits; the fields are processed in chunks).
 * Requires 1 <= lmax < nlat and nlon >= 2 lmax + 1; other shapes, a short workspace and host pointers are refused
 * (SKY_ERR_ARG) before anything is launched.  Asynchronous and stream-ordered; launches on the device that owns x. */
SKY_API size_t sky_grf_workspace_bytes(int32_t members, int32_t channels, int32_t nlat, int32_t nlon, int32_t lmax);
SKY_API int sky_perturb_ic_grf(float* x, const float* sigma_c, float amp, uint64_t seed, int32_t member0, int32_t members,
                       int32_t channels, int32_t nlat, int32_t nlon, int32_t lmax, const float* spec_std,
                       const float* legendre, void* workspace, size_t workspace_bytes, void* stream);
/* The coefficients sky_perturb_ic_grf draws, for inspection: coeffs = device complex64
 * [members * channels][(lmax + 1)(lmax + 2) / 2], (m, l) triangle m-major (entry (m, l) at m (lmax + 1) - m (m - 1) / 2
 * + l - m), each a_lm rounded once from fp64 to fp32. */
SKY_API int sky_grf_draw(float* coeffs, const float* spec_std, uint64_t seed, int32_t member0, int32_t members,
                 int32_t channels, int32_t lmax, void* stream);

/* Ensemble statistics of `members` states on one device, for the selected channels, into caller-owned device buffers:
 *   member m, channel c is the plane x + m * member_stride + c * plane (plane = nlat * nlon floats), c < channel_count;
 *   channels   host int32 [n_sel], 1 <= n_sel <= 128, each in [0, channel_count); the order of the outputs;
 *   quantiles  host fp64 [n_q], 0 <= n_q <= 8, each in [0, 1];
 *   event_sel  host int32 [n_events], 0 <= n_events <= 64: event e is about channels[event_sel[e]]; nondecreasing;
 *   event_thr  host fp32 [n_events], finite thresholds;
 *   stats      device fp32 [2 + n_q][n_sel][plane]: mean, spread, then one plane set per quantile;
 *   prob       device fp32 [n_events][plane] (may be NULL when n_events == 0).
 * Per (selected channel, point), over m < members, in fp64 and rounded once to fp32:
 *   mean    = sum_m x_m / M, summed in member order;
 *   spread  = sqrt(sum_m (x_m - mean)^2 / M) with the unrounded mean: the population standard deviation;
 *   q_j     = numpy.quantile(x, q_j, method="linear"): h = q_j (M - 1), x_(floor h) and x_(ceil h) of the sorted members
 *             linearly interpolated with numpy's lerp;
 *   prob_e  = count(x_m > event_thr[e]) / M (strict: x == t does not count).
 * A NaN member makes every output at that point NaN.  Results are bitwise reproducible (no atomics), a channel's outputs do
 * not depend on which other channels are selected, and quantiles / probabilities do not depend on the member order.
 * Refused with SKY_ERR_ARG before any launch: members outside 1..64, member_stride < channel_count * plane, a channel,
 * quantile, event index or threshold out of range, a decreasing event_sel, too many channels / quantiles / events (all
 * checked before any CUDA call), and x / stats / prob that are not device memory on one device.  Asynchronous and
 * stream-ordered; launches on the device that owns x. */
SKY_API int sky_ensemble_stats(const float* x, int32_t members, int64_t member_stride, int64_t plane, int32_t channel_count,
                       const int32_t* channels, int32_t n_sel, const double* quantiles, int32_t n_q,
                       const int32_t* event_sel, const float* event_thr, int32_t n_events, float* stats, float* prob,
                       void* stream);

/* The statistics of sky_ensemble_stats over members pooled from several sources (the members of several models on one
 * device, each model with its own channel layout):
 *   n_sources      1..4;  host arrays of n_sources entries:
 *   x[k]           device pointer of source k: its member j, channel c is the plane x[k] + j * member_stride[k] + c * plane;
 *   members[k]     >= 1, sum over k at most 64;  member_stride[k] >= channel_count[k] * plane;
 *   channels       host int32 [n_sources][n_sel]: the plane index, in source k, of selected channel s (z500 is a different
 *                  plane in every model; a GraphCast state's new slice is reached through x[k] itself);
 *   quantiles, event_sel, event_thr, stats, prob as for sky_ensemble_stats;
 *   means          device fp32 [n_sources][n_sel][plane] or NULL: the mean of source k's own members.
 * Members are pooled in source-then-member order, so one source gives sky_ensemble_stats' results bit for bit, and means[k]
 * is bitwise sky_ensemble_stats' mean over source k alone.  Same arithmetic, NaN rule, reproducibility and independence of
 * the channel selection as sky_ensemble_stats.  The kernel's parameter block (the per-member pointer table, the channel
 * tables, quantiles and events) is 3336 bytes, inside the 4 KB launch-parameter limit.  Refused with SKY_ERR_ARG before
 * any CUDA call: a count, channel, quantile, event index or threshold out of range, a decreasing event_sel, more than 64
 * members in all; and before any launch: pointers that are not device memory on one device.  Asynchronous and
 * stream-ordered; launches on the device that owns the sources. */
SKY_API int sky_ensemble_stats_multi(int32_t n_sources, const float* const* x, const int32_t* members,
                             const int64_t* member_stride, const int32_t* channel_count, const int32_t* channels,
                             int32_t n_sel, int64_t plane, const double* quantiles, int32_t n_q, const int32_t* event_sel,
                             const float* event_thr, int32_t n_events, float* stats, float* prob, float* means,
                             void* stream);

/* Forecast verification sums of `members` states on one device against an analysis (and optionally a climatology), per
 * latitude-band region and selected channel, into caller-owned device buffers (skyrim_b200/scores.py forms the metrics):
 *   member m, channel c is the plane x + m * member_stride + c * plane (plane = nlat * nlon floats, rows of nlon points
 *              from the northernmost latitude), c < channel_count; members 1..64;
 *   channels     host int32 [n_sel], 1 <= n_sel <= 128, each in [0, channel_count); the order of the outputs;
 *   truth        device fp32 [n_sel][plane]: the analysis of each selected channel (only the selected planes);
 *   clim         device fp32 [n_sel][plane], or NULL: the climatology of each selected channel;
 *   row_weights  device fp64 [n_regions][nlat], 1 <= n_regions <= 4: the weight of every point of row i in region r,
 *                unnormalised, 0 outside the region's band (skyrim_b200.scores.region_weights: cos latitude, poles 0);
 *   partial      device fp64 workspace of at least partial_bytes = 8 * SKY_SCORES_BLOCKS * 9 * n_regions * n_sel bytes;
 *   sums         device fp64 [n_regions][n_sel][9].
 * With M members, x_bar their mean summed in member order in fp64 (the unrounded mean of sky_ensemble_stats), y the truth,
 * k the climatology and w the row weight of a point, the nine sums over the points with w > 0 are
 *   sum w,  sum w e,  sum w e^2  (e = x_bar - y),  sum w sum_m (x_m - x_bar)^2,  sum w (1/M) sum_m |x_m - y|,
 *   sum w G  (G = sum_{m<k} |x_m - x_k|, from the sorted members),  sum w f'o',  sum w f'^2,  sum w o'^2
 *   (f' = x_bar - k, o' = y - k; these three are NaN when clim is NULL).
 * All per-point arithmetic is fp64.  A NaN member, truth or climatology value at a point with w > 0 in a region makes that
 * region's sums 1..8 of that channel NaN; points with w = 0 in a region are not read into its sums.  Two launches, no
 * atomics: each of SKY_SCORES_BLOCKS blocks per channel writes one partial per (region, channel, sum), then the partials
 * are summed in block order, so the sums are bitwise reproducible and a channel's or a region's sums do not depend on the
 * rest of the request.  Refused with SKY_ERR_ARG before any CUDA call: members, nlat, nlon, channel_count, member_stride
 * (< channel_count * plane), a channel, n_sel, n_regions or partial_bytes out of range, null pointers; and before any
 * launch: x, truth, clim, row_weights, partial or sums not device memory on one device.  Asynchronous and stream-ordered;
 * launches on the device that owns x. */
#define SKY_SCORES_BLOCKS 128
SKY_API int sky_forecast_scores(const float* x, int32_t members, int64_t member_stride, int32_t nlat, int32_t nlon,
                                int32_t channel_count, const int32_t* channels, int32_t n_sel, const float* truth,
                                const float* clim, const double* row_weights, int32_t n_regions, double* partial,
                                uint64_t partial_bytes, double* sums, void* stream);

/* Rank histogram (Talagrand diagram) of the truth among `members` states on one device, per latitude-band region and
 * selected channel, into caller-owned device buffers.  x, members, member_stride, nlat, nlon, channel_count, channels,
 * n_sel, truth and row_weights as for sky_forecast_scores;
 *   seed, date_index, lead_index  the Philox key (seed < 2^32, date_index) and the lead word of the tie-breaking draws;
 *   counts       device int32 workspace of at least counts_bytes = 4 * n_sel * nlat * (members + 2) bytes;
 *   hist         device fp64 [n_regions][n_sel][members + 1].
 * At each point, with L = #{x_m < y} and E = #{x_m = y}, the truth's rank is L + floor(u (E + 1)), u = w / 2^32 and w the
 * first output word of Philox4x32-10 at key (seed, date_index), counter (point index in the plane, "RNK1" = 0x524E4B31,
 * channels[s], lead_index): ties are broken at random (Hamill 2001), so a 1-member forecast equal to its truth spreads
 * over both bins instead of filling bin 0.  A point's rank depends on nothing else: not on the channel selection, the
 * regions, the batch or the launch geometry.  hist[r][s][k] = sum over the points with w > 0 of (w / nlon) 1{rank = k},
 * which sums to 1 over k for the normalised weights of skyrim_b200.scores.region_weights.  A NaN member or truth value at
 * a point with w > 0 in a region makes that region's whole histogram of that channel NaN.  Two launches, no atomics on
 * floating-point values: per (row, channel) integer counts per rank, then a sum over the rows in row order, so the
 * histogram is bitwise reproducible and independent of the SM count.  Refused with SKY_ERR_ARG before any CUDA call:
 * the arguments sky_forecast_scores refuses, a seed of 2^32 or more, a negative date_index or lead_index, counts_bytes
 * out of range, null pointers; and before any launch: x, truth, row_weights, counts or hist not device memory on one
 * device.  Asynchronous and stream-ordered; launches on the device that owns x. */
SKY_API int sky_forecast_rank_histogram(const float* x, int32_t members, int64_t member_stride, int32_t nlat, int32_t nlon,
                                        int32_t channel_count, const int32_t* channels, int32_t n_sel, const float* truth,
                                        const double* row_weights, int32_t n_regions, uint64_t seed, int32_t date_index,
                                        int32_t lead_index, int32_t* counts, uint64_t counts_bytes, double* hist,
                                        void* stream);

/* Per-point score-map accumulators of `members` states on one device against an analysis, added in place.
 * x, members, member_stride, nlat, nlon, channel_count, channels, n_sel and truth as for sky_forecast_scores;
 *   maps         device fp64 [n_sel][5][plane], accumulated in place: maps[s][t][p] += term t at point p.
 * The five terms are sky_forecast_scores' sums 1..5 per point instead of summed: e = x_bar - y, e^2,
 * sum_m (x_m - x_bar)^2, (1/M) sum_m |x_m - y| and G = sum_{m<k} |x_m - x_k|, with the same fp64 arithmetic (one shared
 * device function), so bias, RMSE, spread and CRPS maps follow from them as skyrim_b200.scores.metrics_from_sums forms
 * the scalars.  One thread per (channel, point); each call adds once per point, so accumulators summed over calls are
 * bitwise reproducible in call order.  A NaN member or truth value makes only that point's five accumulators NaN.
 * Refused with SKY_ERR_ARG before any CUDA call: the member, grid, channel and truth arguments sky_forecast_scores
 * refuses, a null maps; and before any launch: x, truth or maps not device memory on one device.  Asynchronous and
 * stream-ordered; launches on the device that owns x. */
SKY_API int sky_forecast_score_maps(const float* x, int32_t members, int64_t member_stride, int32_t nlat, int32_t nlon,
                                    int32_t channel_count, const int32_t* channels, int32_t n_sel, const float* truth,
                                    double* maps, void* stream);

/* The three verification entries above over members pooled from several sources (the members of several models on one
 * device, each model with its own channel layout).  In place of (x, members, member_stride, channel_count, channels) they
 * take the source arguments of sky_ensemble_stats_multi:
 *   n_sources      1..4;  host arrays of n_sources entries:
 *   x[k]           device pointer of source k: its member j, channel c is the plane x[k] + j * member_stride[k] + c * plane;
 *   members[k]     >= 1, sum over k (M) at most 64;  member_stride[k] >= channel_count[k] * plane;
 *   channels       host int32 [n_sources][n_sel]: the plane index, in source k, of selected channel s.
 * Everything else (truth, clim, row_weights, n_regions, the workspaces and their sizes, seed / date_index / lead_index and
 * the outputs) is as for the single-source entry, with M the pooled member count: hist is [n_regions][n_sel][M + 1] and
 * counts_bytes at least 4 * n_sel * nlat * (M + 2).
 * Members are pooled in source-then-member order.  Each entry returns, bit for bit, what its single-source entry returns on
 * one contiguous tensor holding the pooled members in that order, laid out in source 0's channel order (x' with member
 * m = the pooled member m, channels' = channels[0]).  That includes the rank histogram's tie-breaking draws: their Philox
 * channel word is channels[0][s], source 0's plane index of the selected channel.  So one source gives the single-source
 * entry's results exactly.  The kernels are the single-source kernels; each block forms the base pointers of its channel's
 * M members once, so the bytes read are the same.  Parameter blocks: 2712 bytes (scores) and 2720 bytes (histogram, maps),
 * inside the 4 KB launch-parameter limit.  Refused with SKY_ERR_ARG before any CUDA call: the source arguments
 * sky_ensemble_stats_multi refuses (a count out of range, a source with no members, more than 64 members in all, a stride
 * below channel_count[k] * plane, a channel outside its source's range, null pointers) and the single-source entry's own
 * grid, region, key and workspace arguments; and before any launch: pointers that are not device memory on one device.
 * Asynchronous and stream-ordered; launches on the device that owns the sources. */
SKY_API int sky_forecast_scores_multi(int32_t n_sources, const float* const* x, const int32_t* members,
                                      const int64_t* member_stride, const int32_t* channel_count, const int32_t* channels,
                                      int32_t n_sel, int32_t nlat, int32_t nlon, const float* truth, const float* clim,
                                      const double* row_weights, int32_t n_regions, double* partial, uint64_t partial_bytes,
                                      double* sums, void* stream);
SKY_API int sky_forecast_rank_histogram_multi(int32_t n_sources, const float* const* x, const int32_t* members,
                                              const int64_t* member_stride, const int32_t* channel_count,
                                              const int32_t* channels, int32_t n_sel, int32_t nlat, int32_t nlon,
                                              const float* truth, const double* row_weights, int32_t n_regions,
                                              uint64_t seed, int32_t date_index, int32_t lead_index, int32_t* counts,
                                              uint64_t counts_bytes, double* hist, void* stream);
SKY_API int sky_forecast_score_maps_multi(int32_t n_sources, const float* const* x, const int32_t* members,
                                          const int64_t* member_stride, const int32_t* channel_count,
                                          const int32_t* channels, int32_t n_sel, int32_t nlat, int32_t nlon,
                                          const float* truth, double* maps, void* stream);

/* Forecasts at sites.  A site table holds, for n_sites sites at (lat[i], lon[i]) in degrees, a 4-entry stencil of flat
 * plane indices and fp64 weights on the equiangular (nlat, nlon) grid of skyrim_b200.timeloop.equiangular_grid (rows from
 * 90 down to -90 degrees, dphi = 180 / (nlat - 1); columns from 0 degrees, dlam = 360 / nlon), computed on the host in
 * fp64, one rounding per operation:
 *   lam' = fmod(lon, 360), plus 360 if negative;  u = lam' / dlam;  j = floor(u);  b = u - j;  j0 = j mod nlon;
 *   j1 = (j0 + 1) mod nlon;  t = (90 - lat) / dphi;
 *   SKY_SITES_BILINEAR: i0 = min(floor(t), nlat - 2), a = t - i0; weights ((1-a)(1-b), (1-a) b, a (1-b), a b) on
 *                       (i0, j0), (i0, j1), (i0 + 1, j0), (i0 + 1, j1);
 *   SKY_SITES_NEAREST:  row floor(t + 0.5), column floor(u + 0.5) mod nlon (longitude distance around the circle, ties to
 *                       the south and the east), weight 1 there and 0 on the three other entries.
 * The table is validated and uploaded to `device` once by sky_sites_create; no index it holds lies outside the plane.
 * Refused with SKY_ERR_ARG before any CUDA call: a lat outside [-90, 90], a non-finite lat or lon, n_sites outside
 * [1, 2^20], nlat < 2, nlon < 1, nlat x nlon >= 2^31, an unknown method, null pointers.  sky_sites_destroy frees the table
 * (NULL is accepted). */
#define SKY_SITES_BILINEAR 0
#define SKY_SITES_NEAREST 1
typedef struct sky_sites sky_sites_t;
SKY_API int sky_sites_create(sky_sites_t** out, const double* lat, const double* lon, int32_t n_sites, int32_t nlat,
                             int32_t nlon, int32_t method, int device);
SKY_API int sky_sites_destroy(sky_sites_t* s);

/* Samples `members` states at the sites of table s, for the selected channels, into a caller-owned device buffer:
 *   x, members, member_stride, channel_count, channels, n_sel as for sky_ensemble_stats, with plane = nlat x nlon of the
 *              table (a GraphCast state's new slice is reached through x itself);
 *   values     device fp32 [members][n_sel][n_sites].
 * Each value is the fp64 sum of the stencil's terms w_k x_k, added in stencil order with no fused multiply-add, starting
 * from 0; entries of weight exactly 0 are not read (a NaN beside a nearest-neighbour site does not reach it); the sum is
 * rounded once to fp32.  A site on a grid point whose coordinates are exact in binary returns that grid value bit for bit
 * under both methods.  sky_ensemble_stats(values, members, n_sel * n_sites, plane = n_sites, n_sel, ...) gives the site
 * statistics.  One thread per (site, channel), sites along threads; any site order.  Refused with SKY_ERR_ARG before any
 * CUDA call: a null table, the member and channel arguments sky_ensemble_stats refuses, a null x or values; and before any
 * launch: x or values not device memory on the table's device.  Asynchronous and stream-ordered. */
SKY_API int sky_sample_sites(const sky_sites_t* s, const float* x, int32_t members, int64_t member_stride,
                             int32_t channel_count, const int32_t* channels, int32_t n_sel, float* values, void* stream);

/* Site verification terms against observations with gaps, into caller-owned device buffers:
 *   values   device fp32 [members][n_sel][n_sites] (sky_sample_sites), members 1..64, n_sel 1..128, n_sites 1..2^20;
 *   obs      device fp32 [n_sel][n_sites]: the observation of each selected channel at each site, NaN where missing;
 *   acc      device fp64 [n_sel][n_sites][6], accumulated in place;
 *   partial  device fp64 workspace of at least partial_bytes = 8 * 6 * n_sel * ceil(n_sites / SKY_SITES_THREADS) bytes;
 *   sums     device fp64 [n_sel][6].
 * At a site with an observation y, with x_bar the members' mean summed in member order in fp64, the six terms are
 *   1,  e = x_bar - y,  e^2,  sum_m (x_m - x_bar)^2,  (1/M) sum_m |x_m - y|,  G = sum_{m<k} |x_m - x_k|,
 * the arithmetic of sky_forecast_score_maps (one shared device function).  acc[s][i][t] += term t once per call (call
 * order, so accumulators summed over calls are bitwise reproducible); sums[s][t] is the sum of term t over the sites of
 * channel s with an observation.  A missing observation adds nothing.  A NaN member at a site with an observation makes
 * terms 1..5 of that site's accumulators and of that channel's sums NaN; term 0 counts the observations.  Two launches,
 * no atomics: one partial per (channel, term, block of SKY_SITES_THREADS sites) summed in thread order, then the partials
 * in block order, so the sums are bitwise reproducible and a channel's results do not depend on the other channels.
 * Refused with SKY_ERR_ARG before any CUDA call: a count or partial_bytes out of range, null pointers; and before any
 * launch: buffers not device memory on one device.  Asynchronous and stream-ordered; launches on the device of values. */
#define SKY_SITES_THREADS 128
SKY_API int sky_site_scores(const float* values, int32_t members, int32_t n_sel, int32_t n_sites, const float* obs,
                            double* acc, double* partial, uint64_t partial_bytes, double* sums, void* stream);

/* Per-kernel-family device timing (CUDA events recorded on the launching stream around the
 * launches whose family bit is set in tag_mask).  profile_end synchronises on the recorded
 * events and returns the summed milliseconds and launch counts per family.  Used by bench.py
 * for the live roofline figure; off by default (no events are recorded). */
SKY_API int sky_model_profile_begin(sky_model_t* m, uint64_t tag_mask);
SKY_API int sky_model_profile_end(sky_model_t* m, double* ms_per_tag, uint64_t* launches_per_tag, int32_t n_tags);
SKY_API int sky_profile_tag_count(void);
SKY_API const char* sky_profile_tag_name(int32_t tag);

/* how many kernels this library has launched since load (bench.py's gpu_launches) */
SKY_API uint64_t sky_launch_count(void);

SKY_API int sky_model_destroy(sky_model_t* m);

#ifdef __cplusplus
}
#endif
#endif /* SKYRIM_B200_H */
