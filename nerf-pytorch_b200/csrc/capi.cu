// capi.cu -- extern "C" entry points of libnerf_b200.so (see include/nerf_b200.h).
#include <stdarg.h>
#include "common.cuh"
#include "small_kernels.cuh"
#include "bwd_simt.cuh"
#include "mlp_simt.cuh"
#include "fused_tc.cuh"
#include "fused_wg.cuh"
#include "bwd_wg.cuh"
#include "train_step.cuh"
#include "mesh.cuh"
#include <stdlib.h>

namespace nb {
#ifdef NERF_B200_PHASE_PROBE
static long long g_phase_launches = 0;      // forward launches since the last nerf_b200_phase_probe_reset
#endif
thread_local char g_err[512] = {0};
long long g_launches = 0;
int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

// ---- optional device-time accounting of the tensor-core kernel launches (bench.py roofline) ----
struct TimedLaunch { cudaEvent_t a, b; double flops; int kind; };   // kind 0: forward pass, 1: dgrad chain, 2: wgrad
static bool g_timing = false;
static TimedLaunch g_timed[4096];
static int g_ntimed = 0;

// the device-time bracket of one launch: NULL when timing is off (or the table is full)
static TimedLaunch* timing_begin(int kind, double flops, cudaStream_t st) {
  if (!g_timing || g_ntimed >= 4096) return nullptr;
  TimedLaunch* tl = &g_timed[g_ntimed++];
  cudaEventCreate(&tl->a); cudaEventCreate(&tl->b);
  tl->flops = flops;
  tl->kind = kind;
  cudaEventRecord(tl->a, st);
  return tl;
}
static void timing_end(TimedLaunch* tl, cudaStream_t st) { if (tl) cudaEventRecord(tl->b, st); }

static double net_macs_per_row(const NerfNetParams& n) {
  // MACs of the reference's Linear layers per sample row (SURVEY Appendix B)
  double m = (double)n.input_ch * n.W;
  for (int i = 1; i < n.D; ++i) m += (double)((n.skip >= 0 && i == n.skip + 1) ? n.W + n.input_ch : n.W) * n.W;
  if (n.use_viewdirs) m += (double)n.W * n.W + n.W + (double)(n.W + n.input_ch_views) * (n.W / 2) + 3.0 * (n.W / 2);
  else m += (double)n.W * n.output_ch;
  return m;
}

static int check_tc_net(const NerfNetParams* net) {
  NB_CHECK_ARG(net != nullptr, "net is NULL");
  NB_CHECK_ARG(net->W == TC_W, "tensor-core path supports netwidth == 256 (got %d); other widths run on the exact path "
               "(precision FP32, set_precision('fp32'))", net->W);
  NB_CHECK_ARG(net->D >= 2 && net->D <= TC_MAXD, "tensor-core path supports 2 <= netdepth <= %d (got %d)", TC_MAXD, net->D);
  NB_CHECK_ARG(net->input_ch >= 3 && net->input_ch <= 63, "input_ch must be in [3,63] (got %d)", net->input_ch);
  NB_CHECK_ARG(net->skip < net->D - 1, "skip layer must be < D-1");
  if (net->use_viewdirs) NB_CHECK_ARG(net->input_ch_views >= 3 && net->input_ch_views <= 63, "input_ch_views must be in [3,63]");
  return 0;
}

// the exact path (mlp_simt_kernel forward, bwd_simt.cuh backward): one thread per output column, so W <= SIMT_THREADS, and
// W a multiple of 4.  A skip after the last layer is refused as the reference fails on it: its heads would receive W + input_ch
// columns, and mlp_simt_kernel never reaches that concatenation.
static int check_exact_net(const NerfNetParams* net) {
  NB_CHECK_ARG(net != nullptr, "net is NULL");
  NB_CHECK_ARG(net->W >= 4 && net->W <= SIMT_THREADS && net->W % 4 == 0,
               "exact path supports netwidth <= %d and a multiple of 4 (got %d)", SIMT_THREADS, net->W);
  NB_CHECK_ARG(net->D >= 1 && net->D <= NERF_B200_MAX_D, "exact path supports 1 <= netdepth <= %d (got %d)", NERF_B200_MAX_D, net->D);
  NB_CHECK_ARG(net->skip < net->D - 1, "skip layer must be < netdepth - 1 (got skip %d, netdepth %d)", net->skip, net->D);
  return 0;
}

static int smem_optin(const void* fn, size_t bytes) {
  NB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

// per-device facts (SM count; which fixed-size kernels already have their > 48 KB shared-memory opt-in): the library may be
// used on several devices of one process, and cudaFuncSetAttribute is per device
struct DeviceState { int sms, n_optin; const void* optin[16]; };
static DeviceState* device_state() {
  static DeviceState st[64];
  static bool init[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!init[dev]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    st[dev].sms = n > 0 ? n : 132;
    st[dev].n_optin = 0;
    cudaGetLastError();
    init[dev] = true;
  }
  return &st[dev];
}
static int num_sms() { return device_state()->sms; }

// the opt-in of a kernel whose shared memory is the same on every launch: once per device.  (Kernels whose shared memory
// follows the arguments opt in on every call.)
static int smem_optin_once(const void* fn, size_t bytes) {
  DeviceState* ds = device_state();
  for (int i = 0; i < ds->n_optin; ++i) if (ds->optin[i] == fn) return 0;
  if (int rc = smem_optin(fn, bytes)) return rc;
  if (ds->n_optin < 16) ds->optin[ds->n_optin++] = fn;
  return 0;
}

// n floats rounded up to 16 bytes: mlp_simt_kernel stores raw as float4, and raw2outputs_bwd_kernel loads it so, so the exact
// path's scratch buffers start on 16-byte boundaries whatever their row counts
static long long round4(long long n) { return (n + 3) & ~3ll; }

// the exact path's MLP (mlp_simt_kernel) over M rows; its shared memory follows the net, so it opts in on every call
static int launch_mlp_simt(const float* pts, const float* dirs, int dir_stride, long long M, int S, const NerfNetParams& net,
                           int L, int Lv, float* raw, const SimtSave& sv, cudaStream_t st) {
  const size_t sm = simt_smem_bytes(net);
  if (int rc = smem_optin((const void*)mlp_simt_kernel, sm)) return rc;
  mlp_simt_kernel<<<cdiv(M, SIMT_ROWS), SIMT_THREADS, sm, st>>>(pts, dirs, dir_stride, M, S, net, L, Lv, raw, sv);
  NB_LAUNCH_OK("mlp_simt_kernel");
  return 0;
}

static bool is_tc(int precision) { return precision == NERF_B200_PREC_TC_FP16 || precision == NERF_B200_PREC_TC_SPLIT; }
static PackLayout pack_layout_for(const NerfNetParams& net, int precision) {
  return precision == NERF_B200_PREC_TC_SPLIT ? make_pack_layout_split(net) : make_pack_layout(net);
}
#define NB_SPLIT_TRAIN_MSG "precision TC_SPLIT trains through the _split entry points (split records, nerf_b200_march_bwd_split) " \
                           "or through the exact backward (nerf_b200_march_bwd)"

// The network half of a fused tensor-core pass over N rays of S samples (march, run_network, density_grid): validates it,
// fills MarchParams' network fields from the packed image of `precision` and plans the persistent grid (whole rays per CTA,
// balanced over the SMs).
static int tc_pass_setup(const NerfNetParams* net, const void* packed, int precision, int L, long long N, int S,
                         MarchParams& p, PackLayout& PL, TilePlan& plan) {
  if (int rc = check_tc_net(net)) return rc;
  NB_CHECK_ARG(packed != nullptr, precision == NERF_B200_PREC_TC_SPLIT ? "packed weights are NULL (call nerf_b200_pack_weights_split)"
                                                                      : "packed weights are NULL (call nerf_b200_pack_weights)");
  NB_CHECK_ARG(N > 0 && S > 0, "empty ray batch must be handled by the caller (N=%lld S=%d)", N, S);
  NB_CHECK_ARG((long long)N * S < (1ll << 40), "batch too large");
  NB_CHECK_ARG(3 + 6 * L == net->input_ch || (L == 0 && net->input_ch == 3), "multires %d does not match input_ch %d", L, net->input_ch);
  plan = make_tile_plan(N, S, num_sms());
  NB_CHECK_ARG((long long)plan.rays_per_cta * S < (1ll << 30), "rays_per_cta * S overflows");
  PL = pack_layout_for(*net, precision);
  const uint8_t* pk = static_cast<const uint8_t*>(packed);
  memset(&p, 0, sizeof(p));
  p.N = N; p.S = S; p.rays_per_cta = plan.rays_per_cta;
  p.chunks = pk + PL.off_chunks;
  p.bias = reinterpret_cast<const float*>(pk + PL.off_bias);
  p.heads = reinterpret_cast<const float*>(pk + PL.off_heads);
  p.D = net->D; p.skip = net->skip; p.use_viewdirs = net->use_viewdirs; p.L = L; p.IC = net->input_ch;
  return 0;
}

// shared launcher of the fused tensor-core pass; `save` != NULL selects the training-mode kernel (EMIT); precision TC_SPLIT runs
// march_split_kernel on the split packed image (nerf_b200_pack_weights_split)
static int launch_march(const float* rays, int ray_stride, const float* z_vals, const float* pts,
                        const float* dirs, int dir_stride, const float* noise, long long N, int S,
                        const NerfNetParams* net, const void* packed, int L, int Lv, int white_bkgd, int do_composite,
                        const NerfPassOut* out, void* workspace, size_t workspace_bytes, const NerfTrainSave* save, const float* vb_pre,
                        cudaStream_t st, int precision = NERF_B200_PREC_TC_FP16) {
  MarchParams p;
  PackLayout PL;
  TilePlan plan;
  if (int rc = tc_pass_setup(net, packed, precision, L, N, S, p, PL, plan)) return rc;
  const uint8_t* pk = static_cast<const uint8_t*>(packed);
  p.rays = rays; p.ray_stride = ray_stride; p.z_vals = z_vals; p.pts = pts; p.noise = noise;
  p.white_bkgd = white_bkgd; p.do_composite = do_composite;
  if (out) p.out = *out;
  TrainSaveDev sv;
  memset(&sv, 0, sizeof(sv));
  if (save) {
    NB_CHECK_ARG(save->act && save->mask, "training-mode save buffers are NULL");
    const size_t rec_act = (precision == NERF_B200_PREC_TC_SPLIT ? 2 : 1) * (size_t)rec_act_bytes(net->D);   // split: hi + lo records
    NB_CHECK_ARG(save->act_bytes >= (size_t)plan.n_tiles * rec_act && save->mask_bytes >= (size_t)plan.n_tiles * rec_mask_bytes(net->D),
                 "training-mode save buffers too small (see nerf_b200_train_record_bytes%s)", precision == NERF_B200_PREC_TC_SPLIT ? "_split" : "");
    NB_CHECK_ARG((reinterpret_cast<uintptr_t>(save->act) & 15) == 0 && (reinterpret_cast<uintptr_t>(save->mask) & 15) == 0, "save buffers must be 16-byte aligned");
    sv.act = static_cast<uint8_t*>(save->act); sv.mask = static_cast<uint8_t*>(save->mask);
    sv.nst_plan = plan.nst; sv.rec_act = (uint32_t)rec_act; sv.rec_mask = rec_mask_bytes(net->D);
  }
  if (net->use_viewdirs && vb_pre != nullptr) {
    p.vb = vb_pre;                                     // the per-ray view-bias table was prepared by ray_setup_kernel
  } else if (net->use_viewdirs) {
    NB_CHECK_ARG(dirs != nullptr, "viewdirs required by a use_viewdirs network");
    NB_CHECK_ARG(workspace != nullptr && workspace_bytes >= (size_t)N * 128 * 4, "workspace too small: need %zu bytes", (size_t)N * 128 * 4);
    NB_CHECK_ARG(3 + 6 * Lv == net->input_ch_views || (Lv == 0 && net->input_ch_views == 3), "multires_views mismatch");
    float* vb = static_cast<float*>(workspace);
    view_bias_kernel<<<cdiv(N, VB_RAYS), 128, 0, st>>>(dirs, dir_stride, N, Lv, net->input_ch_views,
                                                  reinterpret_cast<const float*>(pk + PL.off_vdir), vb);
    NB_LAUNCH_OK("view_bias_kernel");
    p.vb = vb;
  }
  const bool split = precision == NERF_B200_PREC_TC_SPLIT;
  const void* kernel = split ? (save ? (const void*)march_split_train_kernel : (const void*)march_split_kernel) : !save ? (const void*)march_wg_kernel<false> : (const void*)march_wg_kernel<true>;
  if (int rc = smem_optin_once(kernel, FWD_ALLOC)) return rc;
  TimedLaunch* tl = timing_begin(0, 2.0 * net_macs_per_row(*net) * (double)(N * (long long)S), st);
#ifdef NERF_B200_PHASE_PROBE
  {
    const int slot = (int)(g_phase_launches++ % PH_SLOTS);
    NB_CUDA(cudaMemcpyToSymbolAsync(g_fwd_phase_slot, &slot, sizeof(int), 0, cudaMemcpyHostToDevice, st));
  }
#endif
  if (split) {
    const float* wscale = reinterpret_cast<const float*>(pk + PL.off_wscale);
    if (save) march_split_train_kernel<<<plan.grid, TC_THREADS, FWD_ALLOC, st>>>(p, sv, wscale);
    else march_split_kernel<<<plan.grid, TC_THREADS, FWD_ALLOC, st>>>(p, wscale);
    timing_end(tl, st);
    NB_LAUNCH_OK(save ? "march_split_train_kernel" : "march_split_kernel");
    return 0;
  }
  if (save) march_wg_kernel<true><<<plan.grid, TC_THREADS, FWD_ALLOC, st>>>(p, sv);
  else march_wg_kernel<false><<<plan.grid, TC_THREADS, FWD_ALLOC, st>>>(p, sv);
  timing_end(tl, st);
  NB_LAUNCH_OK("march_wg_kernel");
  return 0;
}

// Forward layer l of the packed image: weight [rows][ld], whose first `in` columns are the encoded input (layer 0 and the layer
// after the skip: cat([input_pts, h])) and the next `h` the previous activation.
struct FwdLayer { const float* w; int ld, rows, in, h; };
static FwdLayer fwd_layer(const NerfNetParams& n, int l) {
  const int IC = n.input_ch, W = n.W;
  if (l == 0) return {n.pts_w[0], IC, 256, IC, 0};
  if (l < n.D) {
    const bool sk = n.skip >= 0 && l == n.skip + 1;
    return {n.pts_w[l], sk ? W + IC : W, 256, sk ? IC : 0, W};
  }
  if (l == n.D) return {n.feature_w, W, 256, 0, W};
  return {n.views_w, W + n.input_ch_views, 128, 0, W};                  // the view columns go to the per-ray view bias
}

// The forward's chunks in stream order (K = 32 each: two over the input columns, eight over h), `row_bytes` per row of a chunk
// from PL.off_chunks; layer[i] (if given) receives chunk i's layer.  False when the table disagrees with the layout.
static bool fwd_chunks(const NerfNetParams& n, const PackLayout& PL, unsigned row_bytes, PackJob& job, unsigned char* layer) {
  job.n = 0;
  unsigned off = (unsigned)PL.off_chunks;
  for (int l = 0; l < PL.NL; ++l) {
    const FwdLayer L = fwd_layer(n, l);
    auto add = [&](int k0, int kvalid) {
      if (layer) layer[job.n] = (unsigned char)l;
      PackChunk& c = job.c[job.n++];
      c.src = L.w; c.sn = L.ld; c.sk = 1; c.k0 = k0; c.kvalid = kvalid < 0 ? 0 : (kvalid > 32 ? 32 : kvalid); c.nrows = L.rows; c.dst_off = off;
      off += (unsigned)L.rows * row_bytes;
    };
    if (L.in) { add(0, L.in); add(32, L.in - 32); }
    for (int k0 = L.in; k0 < L.in + L.h; k0 += 32) add(k0, 32);
  }
  return job.n == PL.n_chunks && off == PL.off_chunks + PL.chunk_bytes;
}

// the fp32 tables (biases, heads, view-layer columns) of either image
static int pack_tables(const NerfNetParams& net, const PackLayout& PL, uint8_t* dst, cudaStream_t st) {
  PackTables t;
  t.net = net; t.off_bias = PL.off_bias; t.off_heads = PL.off_heads; t.off_vdir = PL.off_vdir;
  pack_tables_kernel<<<8, 256, 0, st>>>(t, dst);
  NB_LAUNCH_OK("pack_tables_kernel");
  return 0;
}

}  // namespace nb

using namespace nb;

extern "C" {

int nerf_b200_abi_version(void) { return NERF_B200_ABI_VERSION; }
const char* nerf_b200_last_error(void) { return g_err; }
int64_t nerf_b200_launch_count(void) { return g_launches; }

int nerf_b200_timing_enable(int on) { g_timing = on != 0; return 0; }
int nerf_b200_timing_read(double* kernel_ms, int64_t* launches, double* algorithmic_flops) {
  return nerf_b200_timing_read_kinds(kernel_ms, launches, algorithmic_flops, nullptr);
}
// kind_ms[3]: device time of the forward passes, the dgrad chains and the wgrad kernels (NULL: not wanted)
int nerf_b200_timing_read_kinds(double* kernel_ms, int64_t* launches, double* algorithmic_flops, double* kind_ms) {
  double ms = 0, fl = 0, km[3] = {0, 0, 0};
  for (int i = 0; i < g_ntimed; ++i) {
    NB_CUDA(cudaEventSynchronize(g_timed[i].b));
    float t = 0;
    NB_CUDA(cudaEventElapsedTime(&t, g_timed[i].a, g_timed[i].b));
    ms += t; fl += g_timed[i].flops;
    if (g_timed[i].kind >= 0 && g_timed[i].kind < 3) km[g_timed[i].kind] += t;
    cudaEventDestroy(g_timed[i].a); cudaEventDestroy(g_timed[i].b);
  }
  if (kernel_ms) *kernel_ms = ms;
  if (launches) *launches = g_ntimed;
  if (algorithmic_flops) *algorithmic_flops = fl;
  if (kind_ms) { kind_ms[0] = km[0]; kind_ms[1] = km[1]; kind_ms[2] = km[2]; }
  g_ntimed = 0;
  return 0;
}

int nerf_b200_embed(const float* x, int64_t M, int L, float* out, void* stream) {
  NB_CHECK_ARG(x && out, "NULL pointer");
  NB_CHECK_ARG(L >= 0 && L <= 16, "num_freqs out of range");
  if (M == 0) return 0;
  long long total = M * (3 + 6 * L);
  embed_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(x, M, L, out);
  NB_LAUNCH_OK("embed_kernel");
  return 0;
}

size_t nerf_b200_packed_bytes(const NerfNetParams* net) {
  if (!net || check_tc_net(net)) return 0;
  return make_pack_layout(*net).total;
}

int nerf_b200_pack_weights(const NerfNetParams* net, void* packed, size_t packed_bytes, void* stream) {
  if (int rc = check_tc_net(net)) return rc;
  const PackLayout PL = make_pack_layout(*net);
  NB_CHECK_ARG(packed && packed_bytes >= PL.total, "packed buffer too small (%zu < %zu)", packed_bytes, PL.total);
  cudaStream_t st = (cudaStream_t)stream;
  const int IC = net->input_ch, W = net->W;
  PackJob job;
  NB_CHECK_ARG(fwd_chunks(*net, PL, 64, job, nullptr), "internal: chunk table mismatch");
  dim3 grid(4, job.n);
  pack_chunks_kernel<<<grid, 256, 0, st>>>(job, static_cast<uint8_t*>(packed));
  NB_LAUNCH_OK("pack_chunks_kernel");
  if (PL.bwd_bytes) {
    // backward (dgrad) stream, bwd_wg.cuh: chunk [n][k] = W[k0 + k][col0 + n] -- the transposed weights, so that the
    // chain dA_{l-1} = dA_l W_l runs through the forward's operand layouts.  Step 0: views_linears[0].weight[:, :W]
    // (K = W/2), step 1: feature_linear, then pts_linears[D-1] ... [1] restricted to their h columns.  Without view
    // directions the chain starts at step 2 (dA_{D-1} is seeded from output_linear): only the pts-layer chunks.
    PackJob bj2;
    bj2.n = 0;
    unsigned boff = (unsigned)PL.off_bwd;
    auto addT = [&](const float* src, int ld, int col0, int k0) {
      PackChunk& c = bj2.c[bj2.n++];
      c.src = src + col0; c.sn = 1; c.sk = ld; c.k0 = k0; c.kvalid = 32; c.nrows = 256; c.dst_off = boff;
      boff += 256u * 64u;
    };
    if (net->use_viewdirs) {
      for (int c = 0; c < 4; ++c) addT(net->views_w, W + net->input_ch_views, 0, 32 * c);
      for (int c = 0; c < 8; ++c) addT(net->feature_w, W, 0, 32 * c);
    }
    for (int l = net->D - 1; l >= 1; --l) {
      const bool sk = (net->skip >= 0 && l == net->skip + 1);
      for (int c = 0; c < 8; ++c) addT(net->pts_w[l], sk ? W + IC : W, sk ? IC : 0, 32 * c);
    }
    NB_CHECK_ARG(bj2.n == bwd_stream_chunks(net->D, net->use_viewdirs) && boff == PL.off_bwd + PL.bwd_bytes, "internal: backward chunk table mismatch");
    dim3 g2(4, bj2.n);
    pack_chunks_kernel<<<g2, 256, 0, st>>>(bj2, static_cast<uint8_t*>(packed));
    NB_LAUNCH_OK("pack_chunks_kernel (backward stream)");
  }
  return pack_tables(*net, PL, static_cast<uint8_t*>(packed), st);
}

size_t nerf_b200_packed_bytes_split(const NerfNetParams* net) {
  if (!net || check_tc_net(net)) return 0;
  return make_pack_layout_split(*net).total;
}

// the split image (precision TC_SPLIT, fused_tc.cuh: make_pack_layout_split): per-layer weight scales, the forward chunks as
// hi | lo stages of the scaled weights, and the fp16 image's fp32 tables
int nerf_b200_pack_weights_split(const NerfNetParams* net, void* packed, size_t packed_bytes, void* stream) {
  if (int rc = check_tc_net(net)) return rc;
  const PackLayout PL = make_pack_layout_split(*net);
  NB_CHECK_ARG(packed && packed_bytes >= PL.total, "packed buffer too small (%zu < %zu)", packed_bytes, PL.total);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* dst = static_cast<uint8_t*>(packed);
  float* scale = reinterpret_cast<float*>(dst + PL.off_wscale);
  PackSplitJob job;
  memset(&job, 0, sizeof(job));
  NB_CHECK_ARG(fwd_chunks(*net, PL, 128, job.job, job.layer), "internal: split chunk table mismatch");   // hi | lo stages
  SplitScaleJob sj;
  memset(&sj, 0, sizeof(sj));
  sj.n = PL.NL;
  for (int l = 0; l < PL.NL; ++l) {
    const FwdLayer L = fwd_layer(*net, l);
    sj.src[l] = L.w; sj.rows[l] = L.rows; sj.cols[l] = L.in + L.h; sj.ld[l] = L.ld;
  }
  split_scale_kernel<<<PL.NL, 256, 0, st>>>(sj, scale);
  NB_LAUNCH_OK("split_scale_kernel");
  pack_chunks_split_kernel<<<dim3(8, job.job.n), 256, 0, st>>>(job, scale, dst);
  NB_LAUNCH_OK("pack_chunks_split_kernel");
  return pack_tables(*net, PL, dst, st);
}

size_t nerf_b200_packed_bytes_split_train(const NerfNetParams* net) {
  if (!net || check_tc_net(net)) return 0;
  return make_pack_layout_split_train(*net).total;
}

// the split training image (fused_tc.cuh: make_pack_layout_split_train): the split image, then the backward's transposed chunks
// as hi | lo stages of the weights under their layer's scale (the dgrad chain undoes it in its epilogue)
int nerf_b200_pack_weights_split_train(const NerfNetParams* net, void* packed, size_t packed_bytes, void* stream) {
  if (int rc = check_tc_net(net)) return rc;
  const PackLayout PL = make_pack_layout_split_train(*net);
  NB_CHECK_ARG(packed && packed_bytes >= PL.total, "packed buffer too small (%zu < %zu)", packed_bytes, PL.total);
  if (int rc = nerf_b200_pack_weights_split(net, packed, packed_bytes, stream)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* dst = static_cast<uint8_t*>(packed);
  const int IC = net->input_ch, W = net->W, D = net->D;
  PackSplitJob bj;
  memset(&bj, 0, sizeof(bj));
  unsigned boff = (unsigned)PL.off_bwd;
  auto addT = [&](const float* src, int ld, int col0, int k0, int layer) {
    bj.layer[bj.job.n] = (unsigned char)layer;
    PackChunk& c = bj.job.c[bj.job.n++];
    c.src = src + col0; c.sn = 1; c.sk = ld; c.k0 = k0; c.kvalid = 32; c.nrows = 256; c.dst_off = boff;
    boff += 2u * 256u * 64u;
  };
  if (net->use_viewdirs) {
    for (int c = 0; c < 4; ++c) addT(net->views_w, W + net->input_ch_views, 0, 32 * c, D + 1);
    for (int c = 0; c < 8; ++c) addT(net->feature_w, W, 0, 32 * c, D);
  }
  for (int l = D - 1; l >= 1; --l) {
    const bool sk = (net->skip >= 0 && l == net->skip + 1);
    for (int c = 0; c < 8; ++c) addT(net->pts_w[l], sk ? W + IC : W, sk ? IC : 0, 32 * c, l);
  }
  NB_CHECK_ARG(bj.job.n == bwd_stream_chunks(D, net->use_viewdirs) && boff == PL.off_bwd + PL.bwd_bytes, "internal: split backward chunk table mismatch");
  pack_chunks_split_kernel<<<dim3(8, bj.job.n), 256, 0, st>>>(bj, reinterpret_cast<const float*>(dst + PL.off_wscale), dst);
  NB_LAUNCH_OK("pack_chunks_split_kernel (backward stream)");
  return 0;
}

int nerf_b200_run_network(const float* pts, const float* viewdirs, int64_t N, int S, const NerfNetParams* net,
                          const void* packed, int multires, int multires_views, int precision, float* raw,
                          void* workspace, size_t workspace_bytes, void* stream) {
  NB_CHECK_ARG(pts && raw && net, "NULL pointer");
  if (N == 0 || S == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == NERF_B200_PREC_FP32) {
    if (int rc = check_exact_net(net)) return rc;
    NB_CHECK_ARG(!net->use_viewdirs || viewdirs, "viewdirs required");
    return launch_mlp_simt(pts, viewdirs, 3, N * (long long)S, S, *net, multires, multires_views, raw, SimtSave{}, st);
  }
  NB_CHECK_ARG(is_tc(precision), "unknown precision %d", precision);
  NerfPassOut out;
  memset(&out, 0, sizeof(out));
  out.raw = raw;
  return launch_march(nullptr, 0, nullptr, pts, viewdirs, 3, nullptr, N, S, net, packed, multires, multires_views, 0, 0,
                      &out, workspace, workspace_bytes, nullptr, nullptr, st, precision);
}

// ---- mesh extraction ----------------------------------------------------------------------------------------------------
// precision FP32 evaluates the grid in slabs of DENSITY_SLAB points: the points, then mlp_simt_kernel into raw rows, then their
// sigma column.  Workspace: 256 B (the zero view direction every row reads, dir_stride 0) | pts [slab, 3] | raw [slab, 4].
static const long long DENSITY_SLAB = 1ll << 20;

size_t nerf_b200_density_grid_workspace_bytes(int nx, int ny, int nz, const NerfNetParams* net, int precision) {
  if (nx < 1 || ny < 1 || nz < 1) return 0;
  if (precision == NERF_B200_PREC_FP32) {
    if (check_exact_net(net)) return 0;
    const long long P = (long long)nx * ny * nz, slab = P < DENSITY_SLAB ? P : DENSITY_SLAB;
    return 256 + (size_t)round4(slab * 3) * 4 + (size_t)slab * 16;
  }
  if (!is_tc(precision) || check_tc_net(net)) return 0;
  return 256;                                          // the tensor-core pass needs none
}

int nerf_b200_density_grid(const float* xs, int nx, const float* ys, int ny, const float* zs, int nz,
                           const NerfNetParams* net, const void* packed, int multires, int precision,
                           float* sigma, void* workspace, size_t workspace_bytes, void* stream) {
  NB_CHECK_ARG(xs && ys && zs && sigma && net, "NULL pointer");
  NB_CHECK_ARG(nx >= 1 && ny >= 1 && nz >= 1, "empty grid (nx=%d ny=%d nz=%d)", nx, ny, nz);
  NB_CHECK_ARG(precision == NERF_B200_PREC_FP32 || is_tc(precision), "unknown precision %d", precision);
  if (precision == NERF_B200_PREC_FP32) { if (int rc = check_exact_net(net)) return rc; }
  else if (int rc = check_tc_net(net)) return rc;
  NB_CHECK_ARG(3 + 6 * multires == net->input_ch || (multires == 0 && net->input_ch == 3), "multires %d does not match input_ch %d",
               multires, net->input_ch);
  const long long N = (long long)nx * ny, P = N * nz;
  NB_CHECK_ARG(P < (1ll << 40), "grid too large");
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == NERF_B200_PREC_FP32) {
    const size_t need = nerf_b200_density_grid_workspace_bytes(nx, ny, nz, net, precision);
    NB_CHECK_ARG(workspace && workspace_bytes >= need, "workspace too small: need %zu bytes", need);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    const float* zero_dir = reinterpret_cast<const float*>(ws);
    float* pts = reinterpret_cast<float*>(ws + 256);
    const long long slab = P < DENSITY_SLAB ? P : DENSITY_SLAB;
    float* raw = pts + round4(slab * 3);
    NB_CUDA(cudaMemsetAsync(ws, 0, 256, st));
    for (long long m0 = 0; m0 < P; m0 += slab) {
      const long long M = P - m0 < slab ? P - m0 : slab;
      grid_pts_kernel<<<cdiv(M, 256), 256, 0, st>>>(xs, ys, zs, ny, nz, m0, M, pts);
      NB_LAUNCH_OK("grid_pts_kernel");
      if (int rc = launch_mlp_simt(pts, zero_dir, 0, M, 1, *net, multires, 0, raw, SimtSave{}, st)) return rc;
      raw_sigma_kernel<<<cdiv(M, 256), 256, 0, st>>>(raw, M, sigma + m0);
      NB_LAUNCH_OK("raw_sigma_kernel");
    }
    return 0;
  }
  MarchParams p;
  PackLayout PL;
  TilePlan plan;
  if (int rc = tc_pass_setup(net, packed, precision, multires, N, nz, p, PL, plan)) return rc;
  const DensityGrid g{xs, ys, zs, ny, sigma};
  if (precision == NERF_B200_PREC_TC_SPLIT) {
    if (int rc = smem_optin_once((const void*)density_split_kernel, FWD_ALLOC)) return rc;
    density_split_kernel<<<plan.grid, TC_THREADS, FWD_ALLOC, st>>>(p, g, reinterpret_cast<const float*>(static_cast<const uint8_t*>(packed) + PL.off_wscale));
    NB_LAUNCH_OK("density_split_kernel");
  } else {
    if (int rc = smem_optin_once((const void*)density_wg_kernel, FWD_ALLOC)) return rc;
    density_wg_kernel<<<plan.grid, TC_THREADS, FWD_ALLOC, st>>>(p, g);
    NB_LAUNCH_OK("density_wg_kernel");
  }
  return 0;
}

// workspace of marching cubes: McHeader (256 B) | per-point (vertex, face) counts, then offsets [P] | tile sums [P / 4096]
static long long mc_tiles(long long P) { return (P + MC_SCAN_TILE - 1) / MC_SCAN_TILE; }
static size_t mc_need(int nx, int ny, int nz) {
  const long long P = (long long)nx * ny * nz;
  return MC_HEADER_BYTES + (size_t)P * sizeof(int2) + (size_t)mc_tiles(P) * sizeof(int2);
}
// ids and offsets are 32-bit: at most 3 vertices per point and 5 faces per cell
static int check_mc_grid(int nx, int ny, int nz) {
  NB_CHECK_ARG(nx >= 2 && ny >= 2 && nz >= 2, "marching cubes needs nx, ny, nz >= 2 (got %d, %d, %d)", nx, ny, nz);
  const long long P = (long long)nx * ny * nz, Cl = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  NB_CHECK_ARG(3 * P < (1ll << 31) && 5 * Cl < (1ll << 31), "grid of %lld points too large for 32-bit vertex ids", P);
  return 0;
}

size_t nerf_b200_marching_cubes_workspace_bytes(int nx, int ny, int nz) {
  if (check_mc_grid(nx, ny, nz)) return 0;
  return mc_need(nx, ny, nz);
}

int nerf_b200_marching_cubes_count(const float* sigma, int nx, int ny, int nz, float iso, int64_t* counts,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_mc_grid(nx, ny, nz)) return rc;
  NB_CHECK_ARG(sigma && counts && workspace, "NULL pointer");
  const size_t need = mc_need(nx, ny, nz);
  NB_CHECK_ARG(workspace_bytes >= need, "workspace too small: need %zu bytes", need);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const long long P = (long long)nx * ny * nz, nt = mc_tiles(P);
  int2* cnt = reinterpret_cast<int2*>(ws + MC_HEADER_BYTES);
  int2* tsum = cnt + P;
  mc_count_kernel<<<cdiv(P, 256), 256, 0, st>>>(sigma, nx, ny, nz, iso, cnt);
  NB_LAUNCH_OK("mc_count_kernel");
  mc_scan_tiles_kernel<<<(int)nt, MC_SCAN_THREADS, 0, st>>>(cnt, P, tsum);
  NB_LAUNCH_OK("mc_scan_tiles_kernel");
  McHeader h;
  memset(&h, 0, sizeof(h));
  h.nx = nx; h.ny = ny; h.nz = nz; h.iso = iso;
  mc_scan_sums_kernel<<<1, MC_SCAN_THREADS, 0, st>>>(tsum, (int)nt, reinterpret_cast<long long*>(counts), reinterpret_cast<McHeader*>(ws), h);
  NB_LAUNCH_OK("mc_scan_sums_kernel");
  mc_scan_add_kernel<<<cdiv(P, 256), 256, 0, st>>>(cnt, P, tsum);
  NB_LAUNCH_OK("mc_scan_add_kernel");
  return 0;
}

int nerf_b200_marching_cubes_emit(const float* sigma, const float* xs, const float* ys, const float* zs,
                                  int nx, int ny, int nz, float iso, float* verts, int64_t max_verts,
                                  int32_t* faces, int64_t max_faces, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  if (int rc = check_mc_grid(nx, ny, nz)) return rc;
  NB_CHECK_ARG(sigma && xs && ys && zs && workspace, "NULL pointer");
  NB_CHECK_ARG((verts || max_verts == 0) && (faces || max_faces == 0) && max_verts >= 0 && max_faces >= 0, "NULL output with a capacity");
  const size_t need = mc_need(nx, ny, nz);
  NB_CHECK_ARG(workspace_bytes >= need, "workspace too small: need %zu bytes", need);
  cudaStream_t st = (cudaStream_t)stream;
  McHeader h;
  NB_CUDA(cudaMemcpyAsync(&h, workspace, sizeof(h), cudaMemcpyDeviceToHost, st));
  NB_CUDA(cudaStreamSynchronize(st));
  NB_CHECK_ARG(h.nx == nx && h.ny == ny && h.nz == nz && memcmp(&h.iso, &iso, sizeof(float)) == 0,
               "the workspace holds the counts of another grid or iso (call nerf_b200_marching_cubes_count first)");
  NB_CHECK_ARG(max_verts >= h.V && max_faces >= h.F, "outputs too small: %lld vertices and %lld faces need room (got %lld, %lld)",
               h.V, h.F, (long long)max_verts, (long long)max_faces);
  const long long P = (long long)nx * ny * nz;
  mc_emit_kernel<<<cdiv(P, 256), 256, 0, st>>>(sigma, xs, ys, zs, nx, ny, nz, iso,
                                                reinterpret_cast<const int2*>(static_cast<uint8_t*>(workspace) + MC_HEADER_BYTES), verts, faces);
  NB_LAUNCH_OK("mc_emit_kernel");
  return 0;
}

int nerf_b200_raw2outputs(const float* raw, const float* z_vals, const float* rays_d, int d_stride, const float* noise,
                          int64_t N, int S, int white_bkgd, const NerfPassOut* out, void* stream) {
  NB_CHECK_ARG(raw && z_vals && rays_d && out, "NULL pointer");
  NB_CHECK_ARG(S >= 1, "S must be >= 1");
  if (N == 0) return 0;
  raw2outputs_kernel<<<cdiv(N * 32, 256), 256, 0, (cudaStream_t)stream>>>(raw, z_vals, rays_d, d_stride, noise, N, S, white_bkgd, *out);
  NB_LAUNCH_OK("raw2outputs_kernel");
  return 0;
}

}  // extern "C"

static NerfOutGrads rgb_seed(const float* g_rgb) {
  NerfOutGrads g;
  memset(&g, 0, sizeof(g));
  g.rgb_map = g_rgb;
  return g;
}
static bool seeds_rgb_only(const NerfOutGrads& g) { return !(g.disp_map || g.acc_map || g.depth_map || g.weights || g.raw); }
static bool seeds_none(const NerfOutGrads& g) { return !g.rgb_map && seeds_rgb_only(g); }
// the seeds of rays [n0, n0 + nn) of a pass with S samples per ray
static NerfOutGrads seeds_at(const NerfOutGrads& g, int64_t n0, int S) {
  NerfOutGrads o = g;
  const long long nS = n0 * (long long)S;
  if (o.rgb_map) o.rgb_map += n0 * 3;
  if (o.disp_map) o.disp_map += n0;
  if (o.acc_map) o.acc_map += n0;
  if (o.depth_map) o.depth_map += n0;
  if (o.weights) o.weights += nS;
  if (o.raw) o.raw += nS * 4;
  return o;
}

// the compositing adjoint for any set of seeds.  rgb_map alone without `amax`: the rgb-only instantiation (the library's
// original arithmetic); otherwise the seeded one, which with `amax` also forms the loss-scale input of the pass.
static int raw2outputs_bwd_impl(const float* raw, const float* z_vals, const float* rays_d, int d_stride, const float* noise,
                                int64_t N, int S, int white_bkgd, const NerfOutGrads& g, unsigned int* amax, float* d_raw,
                                cudaStream_t st) {
  NB_CHECK_ARG(raw && z_vals && rays_d && d_raw, "NULL pointer");
  NB_CHECK_ARG(!seeds_none(g), "no output gradient given (every NerfOutGrads member is NULL)");
  NB_CHECK_ARG(S >= 1 && S <= 1024, "S must be in [1,1024]");
  if (N == 0) return 0;
  const int wpb = 4;
  const size_t sm = (size_t)wpb * 4 * S * sizeof(float);
  R2OSeeds s = {g.rgb_map, g.disp_map, g.acc_map, g.depth_map, g.weights, g.raw, amax};
  if (seeds_rgb_only(g) && !amax) {
    if (int rc = smem_optin((const void*)raw2outputs_bwd_kernel<false>, sm)) return rc;
    raw2outputs_bwd_kernel<false><<<cdiv(N, wpb), wpb * 32, sm, st>>>(raw, z_vals, rays_d, d_stride, noise, N, S, white_bkgd, s, d_raw);
  } else {
    if (int rc = smem_optin((const void*)raw2outputs_bwd_kernel<true>, sm)) return rc;
    raw2outputs_bwd_kernel<true><<<cdiv(N, wpb), wpb * 32, sm, st>>>(raw, z_vals, rays_d, d_stride, noise, N, S, white_bkgd, s, d_raw);
  }
  NB_LAUNCH_OK("raw2outputs_bwd_kernel");
  return 0;
}

extern "C" {

int nerf_b200_raw2outputs_bwd(const float* raw, const float* z_vals, const float* rays_d, int d_stride, const float* noise,
                              int64_t N, int S, int white_bkgd, const float* g_rgb, float* d_raw, void* stream) {
  return raw2outputs_bwd_impl(raw, z_vals, rays_d, d_stride, noise, N, S, white_bkgd, rgb_seed(g_rgb), nullptr, d_raw, (cudaStream_t)stream);
}

int nerf_b200_raw2outputs_bwd_outs(const float* raw, const float* z_vals, const float* rays_d, int d_stride, const float* noise,
                                   int64_t N, int S, int white_bkgd, const NerfOutGrads* g, float* d_raw, void* stream) {
  NB_CHECK_ARG(g, "NULL pointer");
  return raw2outputs_bwd_impl(raw, z_vals, rays_d, d_stride, noise, N, S, white_bkgd, *g, nullptr, d_raw, (cudaStream_t)stream);
}

static int fill_pack_args(PackRaysArgs& a, const float* rays_o, const float* rays_d, const float* view_src, const NerfCamera* cam, int64_t N,
                          int64_t pixel0, const int64_t* pixel_index, int ndc, float near, float far, int use_viewdirs) {
  NB_CHECK_ARG((rays_o && rays_d) || (cam && !rays_o && !rays_d), "give rays_o and rays_d, or a camera to generate them");
  NB_CHECK_ARG(!ndc || cam, "ndc needs the camera (H, W, focal)");
  memset(&a, 0, sizeof(a));
  a.rays_o = rays_o; a.rays_d = rays_d; a.view_src = view_src; a.N = N; a.pixel0 = pixel0;
  a.pixel_index = reinterpret_cast<const long long*>(pixel_index);
  a.ndc = ndc; a.use_viewdirs = use_viewdirs; a.stride = use_viewdirs ? 11 : 8; a.near = near; a.far = far;
  if (cam) {
    a.H = cam->H; a.W = cam->W; a.fx = cam->fx; a.fy = cam->fy; a.cx = cam->cx; a.cy = cam->cy;
    memcpy(a.c2w, cam->c2w, sizeof(a.c2w));
    a.ndc_cw = (float)(-1.0 / ((double)cam->W / (2.0 * (double)cam->fx)));      // run_nerf_helpers.py:181 (focal = K[0][0])
    a.ndc_ch = (float)(-1.0 / ((double)cam->H / (2.0 * (double)cam->fx)));
  }
  return 0;
}

static int pack_rays_impl(const float* rays_o, const float* rays_d, const float* view_src, const NerfCamera* cam, int64_t N,
                          int64_t pixel0, const int64_t* pixel_index, int ndc, float near, float far, int use_viewdirs, float* out, void* stream) {
  NB_CHECK_ARG(out != nullptr, "NULL output");
  if (N == 0) return 0;
  PackRaysArgs a;
  if (int rc = fill_pack_args(a, rays_o, rays_d, view_src, cam, N, pixel0, pixel_index, ndc, near, far, use_viewdirs)) return rc;
  pack_rays_kernel<<<cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(a, out);
  NB_LAUNCH_OK("pack_rays_kernel");
  return 0;
}

int nerf_b200_pack_rays(const float* rays_o, const float* rays_d, const float* view_src, const NerfCamera* cam, int64_t N,
                        int64_t pixel0, int ndc, float near, float far, int use_viewdirs, float* out, void* stream) {
  return pack_rays_impl(rays_o, rays_d, view_src, cam, N, pixel0, nullptr, ndc, near, far, use_viewdirs, out, stream);
}

// the same for an arbitrary list of pixels of the camera's image (the per-image random pixel choice of run_nerf.py:728-757,
// without materialising get_rays' [H, W, 3] tensors or gathering from them)
int nerf_b200_pack_rays_pixels(const NerfCamera* cam, const int64_t* pixel_index, int64_t N, int ndc, float near, float far,
                               int use_viewdirs, float* out, void* stream) {
  NB_CHECK_ARG(cam && pixel_index, "camera and pixel_index are required");
  return pack_rays_impl(nullptr, nullptr, nullptr, cam, N, 0, pixel_index, ndc, near, far, use_viewdirs, out, stream);
}

int nerf_b200_to8b(const float* x, int64_t n, uint8_t* out, void* stream) {
  NB_CHECK_ARG(x && out, "NULL pointer");
  if (n == 0) return 0;
  to8b_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(x, n, out);
  NB_LAUNCH_OK("to8b_kernel");
  return 0;
}

int nerf_b200_sample_pdf(const float* bins, const float* weights, const float* u, int64_t u_row_stride, int64_t N, int B,
                         int n_samples, float* samples, void* stream) {
  NB_CHECK_ARG(bins && weights && u && samples, "NULL pointer");
  NB_CHECK_ARG(B >= 2 && B <= 2048 && n_samples >= 1, "bad B / n_samples");
  if (N == 0) return 0;
  const int wpb = 4;
  const size_t sm = (size_t)wpb * 3 * B * sizeof(float);
  if (int rc = smem_optin((const void*)sample_pdf_kernel, sm)) return rc;
  sample_pdf_kernel<<<cdiv(N, wpb), wpb * 32, sm, (cudaStream_t)stream>>>(bins, weights, u, u_row_stride, N, B, n_samples, samples);
  NB_LAUNCH_OK("sample_pdf_kernel");
  return 0;
}

int nerf_b200_coarse_z(const float* rays, int ray_stride, const float* t_vals, const float* t_rand, int64_t N, int S,
                       int lindisp, float* z_vals, void* stream) {
  NB_CHECK_ARG(rays && t_vals && z_vals, "NULL pointer");
  NB_CHECK_ARG(ray_stride >= 8, "ray_stride must be >= 8");
  if (N == 0) return 0;
  coarse_z_kernel<<<cdiv(N * S, 256), 256, 0, (cudaStream_t)stream>>>(rays, ray_stride, t_vals, t_rand, N, S, lindisp, z_vals);
  NB_LAUNCH_OK("coarse_z_kernel");
  return 0;
}

int nerf_b200_fine_z(const float* z_vals, const float* weights, const float* u, int64_t u_row_stride, int64_t N, int S,
                     int n_imp, float* z_fine, float* z_samples, float* z_std, void* stream) {
  NB_CHECK_ARG(z_vals && weights && u && z_fine, "NULL pointer");
  NB_CHECK_ARG(S >= 3 && n_imp >= 1 && S + n_imp <= 4096, "bad S / n_imp");   // S = 2: the reference fails too (empty cdf)
  if (N == 0) return 0;
  int P = 1;
  while (P < S + n_imp) P <<= 1;
  // four warps (rays) per block, fewer where their rows would pass the opt-in shared-memory limit (from S ~ 3478 at P = 4096)
  int dev = 0, optin = 0;
  NB_CUDA(cudaGetDevice(&dev));
  NB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t row_bytes = (size_t)(3 * S + P) * sizeof(float);
  int wpb = 4;
  while (wpb > 1 && (size_t)wpb * row_bytes > (size_t)optin) --wpb;
  const size_t sm = (size_t)wpb * row_bytes;
  if (int rc = smem_optin((const void*)fine_z_kernel, sm)) return rc;
  fine_z_kernel<<<cdiv(N, wpb), wpb * 32, sm, (cudaStream_t)stream>>>(z_vals, weights, u, u_row_stride, N, S, n_imp, P, z_fine, z_samples, z_std);
  NB_LAUNCH_OK("fine_z_kernel");
  return 0;
}

size_t nerf_b200_march_workspace_bytes(int64_t N, int S) {
  size_t tc = (size_t)N * 128 * 4 * 2, exact = (size_t)N * S * 28;   // view-bias tables of both nets | pts + raw scratch
  return (tc > exact ? tc : exact) + 256;
}

static int march_impl(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                      const void* packed, const NerfRenderCfg* cfg, const NerfPassOut* out, void* workspace,
                      size_t workspace_bytes, const NerfTrainSave* save, void* stream, const float* vb_pre = nullptr) {
  NB_CHECK_ARG(rays && z_vals && net && cfg && out, "NULL pointer");
  if (N == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  NB_CHECK_ARG(cfg->ray_stride >= (net->use_viewdirs ? 11 : 8), "ray_stride %d too small", cfg->ray_stride);
  if (cfg->precision == NERF_B200_PREC_FP32) {
    // exact mode (validation path): materialise pts -> fp32 CUDA-core MLP -> raw2outputs kernel
    NB_CHECK_ARG(save == nullptr, "training-mode records belong to the tensor-core path");
    if (int rc = check_exact_net(net)) return rc;
    const long long M = N * (long long)S;
    const size_t pts_floats = round4(M * 3);
    const size_t need = pts_floats * 4 + (out->raw ? 0 : (size_t)M * 16);
    NB_CHECK_ARG(workspace && workspace_bytes >= need, "exact-mode workspace too small: need %zu bytes", need);
    float* pts = static_cast<float*>(workspace);
    float* raw = out->raw ? out->raw : pts + pts_floats;
    pts_kernel<<<cdiv(M, 256), 256, 0, st>>>(rays, cfg->ray_stride, z_vals, M, S, pts);
    NB_LAUNCH_OK("pts_kernel");
    if (int rc = launch_mlp_simt(pts, rays + 8, cfg->ray_stride, M, S, *net, cfg->multires, cfg->multires_views, raw, SimtSave{}, st)) return rc;
    raw2outputs_kernel<<<cdiv(N * 32, 256), 256, 0, st>>>(raw, z_vals, rays + 3, cfg->ray_stride, noise, N, S, cfg->white_bkgd, *out);
    NB_LAUNCH_OK("raw2outputs_kernel");
    return 0;
  }
  NB_CHECK_ARG(is_tc(cfg->precision), "unknown precision %d", cfg->precision);
  return launch_march(rays, cfg->ray_stride, z_vals, nullptr, rays + 8, cfg->ray_stride, noise, N, S, net, packed,
                      cfg->multires, cfg->multires_views, cfg->white_bkgd, 1, out, workspace, workspace_bytes, save, vb_pre, st,
                      cfg->precision);
}

int nerf_b200_march(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                    const void* packed, const NerfRenderCfg* cfg, const NerfPassOut* out, void* workspace,
                    size_t workspace_bytes, void* stream) {
  return march_impl(rays, z_vals, noise, N, S, net, packed, cfg, out, workspace, workspace_bytes, nullptr, stream);
}

// training mode of one pass: it also leaves the per-tile records of the tensor-core backward (split: the hi + lo records of
// march_split_train_kernel for nerf_b200_march_bwd_split); `split` picks the precision the entry point takes
static int march_train_impl(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                            const void* packed, const NerfRenderCfg* cfg, const NerfPassOut* out, void* workspace,
                            size_t workspace_bytes, const NerfTrainSave* save, void* stream, bool split) {
  NB_CHECK_ARG(save != nullptr && out && out->raw, "training mode needs the save buffers and out->raw (the compositing adjoint reads raw)");
  if (split) NB_CHECK_ARG(cfg && cfg->precision == NERF_B200_PREC_TC_SPLIT, "the split training forward needs precision TC_SPLIT");
  else NB_CHECK_ARG(!cfg || cfg->precision != NERF_B200_PREC_TC_SPLIT, NB_SPLIT_TRAIN_MSG);
  return march_impl(rays, z_vals, noise, N, S, net, packed, cfg, out, workspace, workspace_bytes, save, stream);
}

int nerf_b200_march_train(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                          const void* packed, const NerfRenderCfg* cfg, const NerfPassOut* out, void* workspace,
                          size_t workspace_bytes, const NerfTrainSave* save, void* stream) {
  return march_train_impl(rays, z_vals, noise, N, S, net, packed, cfg, out, workspace, workspace_bytes, save, stream, false);
}

int nerf_b200_march_train_split(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                                const void* packed, const NerfRenderCfg* cfg, const NerfPassOut* out, void* workspace,
                                size_t workspace_bytes, const NerfTrainSave* save, void* stream) {
  return march_train_impl(rays, z_vals, noise, N, S, net, packed, cfg, out, workspace, workspace_bytes, save, stream, true);
}

int nerf_b200_train_record_bytes_split(int64_t N, int S, const NerfNetParams* net, size_t* act_bytes, size_t* mask_bytes) {
  if (int rc = nerf_b200_train_record_bytes(N, S, net, act_bytes, mask_bytes)) return rc;
  if (act_bytes) *act_bytes *= 2;
  return 0;
}

int nerf_b200_train_record_bytes(int64_t N, int S, const NerfNetParams* net, size_t* act_bytes, size_t* mask_bytes) {
  if (int rc = check_tc_net(net)) return rc;
  NB_CHECK_ARG(N >= 0 && S >= 1, "bad N / S");
  const TilePlan plan = make_tile_plan(N > 0 ? N : 1, S, num_sms());
  if (act_bytes) *act_bytes = (size_t)plan.n_tiles * rec_act_bytes(net->D);
  if (mask_bytes) *mask_bytes = (size_t)plan.n_tiles * rec_mask_bytes(net->D);
  return 0;
}

static int render_rays_fwd_impl(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfNetParams* net_coarse,
                                const void* packed_coarse, const NerfNetParams* net_fine, const void* packed_fine,
                                const float* t_vals, const float* u_det, const float* t_rand, const float* u_rand,
                                const float* noise0, const float* noise1, float* z_coarse, const NerfPassOut* coarse,
                                float* z_fine, float* z_std, const NerfPassOut* fine, void* workspace,
                                size_t workspace_bytes, const NerfTrainSave* save_coarse, const NerfTrainSave* save_fine, void* stream,
                                const NerfRayGen* gen = nullptr) {
  NB_CHECK_ARG(rays && cfg && net_coarse && t_vals && z_coarse && coarse, "NULL pointer");
  if (N == 0) return 0;
  // gen: `rays` is still to be built (render()'s batch construction, run_nerf.py:95-123) -- by the prologue kernel below on the
  // tensor-core path, by pack_rays_kernel otherwise
  PackRaysArgs pk;
  bool pack_pending = false;
  if (gen) {
    NB_CHECK_ARG(cfg->ray_stride == (gen->use_viewdirs ? 11 : 8), "ray_stride does not match the batch to build");
    if (int rc = fill_pack_args(pk, gen->rays_o, gen->rays_d, gen->view_src, gen->cam, N, gen->pixel0, nullptr, gen->ndc, gen->near, gen->far, gen->use_viewdirs)) return rc;
    pack_pending = true;
  }
  const int Sc = cfg->N_samples, Ni = cfg->N_importance;
  NB_CHECK_ARG(Sc >= 1 && Ni >= 0, "bad sample counts");
  if (cfg->precision == NERF_B200_PREC_FP32) {          // both nets are checked before the first launch
    if (int rc = check_exact_net(net_coarse)) return rc;
    if (Ni > 0 && net_fine) { if (int rc = check_exact_net(net_fine)) return rc; }
  }
  NB_CHECK_ARG(!cfg->perturb || t_rand, "perturb > 0 needs t_rand");
  // per-ray prologue: z sampling (run_nerf.py:357-379) and, on the tensor-core path, the view-bias tables of both networks
  // -- one launch (ray_setup_kernel); the exact path keeps the stand-alone z kernel
  const NerfNetParams* nf = net_fine ? net_fine : net_coarse;
  const void* pf = net_fine ? packed_fine : packed_coarse;
  const float* vb_c = nullptr;
  const float* vb_f = nullptr;
  if (is_tc(cfg->precision) && net_coarse->use_viewdirs && packed_coarse && (Ni == 0 || (nf->use_viewdirs && pf))) {
    if (int rc = check_tc_net(net_coarse)) return rc;
    NB_CHECK_ARG(workspace != nullptr && workspace_bytes >= (size_t)N * 128 * 4 * 2, "workspace too small: need %zu bytes", (size_t)N * 128 * 4 * 2);
    NB_CHECK_ARG(cfg->ray_stride >= 11, "ray_stride %d too small for view directions", cfg->ray_stride);
    NB_CHECK_ARG(3 + 6 * cfg->multires_views == net_coarse->input_ch_views || (cfg->multires_views == 0 && net_coarse->input_ch_views == 3), "multires_views mismatch");
    const PackLayout PLc = pack_layout_for(*net_coarse, cfg->precision);
    RaySetupArgs a;
    memset(&a, 0, sizeof(a));
    a.rays = rays; a.ray_stride = cfg->ray_stride; a.N = N; a.Lv = cfg->multires_views; a.ICV = net_coarse->input_ch_views;
    float* vb = static_cast<float*>(workspace);
    a.vdir_a = reinterpret_cast<const float*>(static_cast<const uint8_t*>(packed_coarse) + PLc.off_vdir); a.vb_a = vb;
    vb_c = vb;
    if (Ni > 0) {
      if (nf == net_coarse || pf == packed_coarse) vb_f = vb_c;
      else {
        NB_CHECK_ARG(nf->input_ch_views == net_coarse->input_ch_views, "coarse and fine networks must encode view directions alike");
        const PackLayout PLf = pack_layout_for(*nf, cfg->precision);
        a.vdir_b = reinterpret_cast<const float*>(static_cast<const uint8_t*>(pf) + PLf.off_vdir); a.vb_b = vb + (size_t)N * 128;
        vb_f = a.vb_b;
      }
    }
    a.t_vals = t_vals; a.t_rand = cfg->perturb ? t_rand : nullptr; a.S = Sc; a.lindisp = cfg->lindisp; a.z_out = z_coarse;
    if (pack_pending) { a.pack = pk; a.pack_out = const_cast<float*>(rays); pack_pending = false; }
    ray_setup_kernel<<<cdiv(N, VB_RAYS), 256, 0, (cudaStream_t)stream>>>(a);
    NB_LAUNCH_OK("ray_setup_kernel");
  } else {
    if (pack_pending) {
      pack_rays_kernel<<<cdiv(N, 256), 256, 0, (cudaStream_t)stream>>>(pk, const_cast<float*>(rays));
      NB_LAUNCH_OK("pack_rays_kernel");
    }
    if (int rc = nerf_b200_coarse_z(rays, cfg->ray_stride, t_vals, cfg->perturb ? t_rand : nullptr, N, Sc, cfg->lindisp, z_coarse, stream)) return rc;
  }
  // coarse pass (:381-386)
  if (int rc = march_impl(rays, z_coarse, noise0, N, Sc, net_coarse, packed_coarse, cfg, coarse, workspace, workspace_bytes, save_coarse, stream, vb_c)) return rc;
  if (Ni == 0) return 0;
  NB_CHECK_ARG(coarse->weights && z_fine && fine, "N_importance > 0 needs coarse->weights, z_fine and fine outputs");
  // hierarchical sampling (:392-396, :412); det <=> perturb == 0 (:393)
  const float* u = cfg->perturb ? u_rand : u_det;
  NB_CHECK_ARG(u != nullptr, "missing u (u_det for perturb==0, u_rand otherwise)");
  if (int rc = nerf_b200_fine_z(z_coarse, coarse->weights, u, cfg->perturb ? Ni : 0, N, Sc, Ni, z_fine, nullptr, z_std, stream)) return rc;
  // fine pass on all S_c + N_importance samples (:397-403); network_fine None -> coarse net (:399)
  return march_impl(rays, z_fine, noise1, N, Sc + Ni, nf, pf, cfg, fine, workspace, workspace_bytes, save_fine, stream, vb_f);
}

int nerf_b200_render_rays_fwd(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfNetParams* net_coarse,
                              const void* packed_coarse, const NerfNetParams* net_fine, const void* packed_fine,
                              const float* t_vals, const float* u_det, const float* t_rand, const float* u_rand,
                              const float* noise0, const float* noise1, float* z_coarse, const NerfPassOut* coarse,
                              float* z_fine, float* z_std, const NerfPassOut* fine, void* workspace,
                              size_t workspace_bytes, void* stream) {
  return render_rays_fwd_impl(rays, N, cfg, net_coarse, packed_coarse, net_fine, packed_fine, t_vals, u_det, t_rand, u_rand, noise0, noise1,
                              z_coarse, coarse, z_fine, z_std, fine, workspace, workspace_bytes, nullptr, nullptr, stream);
}

// render() for one chunk: the ray batch is BUILT (get_rays / viewdirs / NDC / near-far / packing, run_nerf.py:95-123) by the same
// prologue launch that samples z and fills the view-bias tables, into `rays` [N, 8 | 11], then rendered as above
int nerf_b200_render_fwd(const NerfRayGen* gen, float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfNetParams* net_coarse,
                         const void* packed_coarse, const NerfNetParams* net_fine, const void* packed_fine,
                         const float* t_vals, const float* u_det, const float* t_rand, const float* u_rand,
                         const float* noise0, const float* noise1, float* z_coarse, const NerfPassOut* coarse,
                         float* z_fine, float* z_std, const NerfPassOut* fine, void* workspace,
                         size_t workspace_bytes, void* stream) {
  NB_CHECK_ARG(gen != nullptr, "NULL ray generator");
  return render_rays_fwd_impl(rays, N, cfg, net_coarse, packed_coarse, net_fine, packed_fine, t_vals, u_det, t_rand, u_rand, noise0, noise1,
                              z_coarse, coarse, z_fine, z_std, fine, workspace, workspace_bytes, nullptr, nullptr, stream, gen);
}

// the same call in training mode: both passes also leave their per-tile records (activation images + ReLU masks) for
// the tensor-core backward, and must write raw (coarse->raw, fine->raw).  The refusals of both training entries; `split`
// picks the precision the entry takes.
static int check_fwd_train(const NerfRenderCfg* cfg, const NerfPassOut* coarse, const NerfPassOut* fine,
                           const NerfTrainSave* save_coarse, const NerfTrainSave* save_fine, bool split) {
  if (split) NB_CHECK_ARG(cfg && cfg->precision == NERF_B200_PREC_TC_SPLIT, "the split training forward needs precision TC_SPLIT");
  else {
    NB_CHECK_ARG(cfg && cfg->precision != NERF_B200_PREC_TC_SPLIT, NB_SPLIT_TRAIN_MSG);
    NB_CHECK_ARG(cfg->precision == NERF_B200_PREC_TC_FP16, "training-mode records belong to the tensor-core path");
  }
  NB_CHECK_ARG(save_coarse && coarse && coarse->raw, "training mode needs save_coarse and coarse->raw");
  NB_CHECK_ARG(cfg->N_importance == 0 || (save_fine && fine && fine->raw), "training mode needs save_fine and fine->raw");
  return 0;
}

int nerf_b200_render_rays_fwd_train(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfNetParams* net_coarse,
                                    const void* packed_coarse, const NerfNetParams* net_fine, const void* packed_fine,
                                    const float* t_vals, const float* u_det, const float* t_rand, const float* u_rand,
                                    const float* noise0, const float* noise1, float* z_coarse, const NerfPassOut* coarse,
                                    float* z_fine, float* z_std, const NerfPassOut* fine, void* workspace,
                                    size_t workspace_bytes, const NerfTrainSave* save_coarse, const NerfTrainSave* save_fine, void* stream) {
  if (int rc = check_fwd_train(cfg, coarse, fine, save_coarse, save_fine, false)) return rc;
  return render_rays_fwd_impl(rays, N, cfg, net_coarse, packed_coarse, net_fine, packed_fine, t_vals, u_det, t_rand, u_rand, noise0, noise1,
                              z_coarse, coarse, z_fine, z_std, fine, workspace, workspace_bytes, save_coarse, save_fine, stream);
}

int nerf_b200_render_rays_fwd_train_split(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfNetParams* net_coarse,
                                          const void* packed_coarse, const NerfNetParams* net_fine, const void* packed_fine,
                                          const float* t_vals, const float* u_det, const float* t_rand, const float* u_rand,
                                          const float* noise0, const float* noise1, float* z_coarse, const NerfPassOut* coarse,
                                          float* z_fine, float* z_std, const NerfPassOut* fine, void* workspace,
                                          size_t workspace_bytes, const NerfTrainSave* save_coarse, const NerfTrainSave* save_fine, void* stream) {
  if (int rc = check_fwd_train(cfg, coarse, fine, save_coarse, save_fine, true)) return rc;
  return render_rays_fwd_impl(rays, N, cfg, net_coarse, packed_coarse, net_fine, packed_fine, t_vals, u_det, t_rand, u_rand, noise0, noise1,
                              z_coarse, coarse, z_fine, z_std, fine, workspace, workspace_bytes, save_coarse, save_fine, stream);
}

// ---- exact-mode backward of one pass (see bwd_simt.cuh) -------------------------------------------
static const int BWD_RAYS_PER_SLAB = 512;     // rays recomputed + back-propagated per slab (bounds the workspace)

// march_bwd_impl carves BWD_BUFFERS buffers per slab, each rounded up to 4 floats: the 1024 spare bytes cover the rounding
static const int BWD_BUFFERS = 11;
static_assert(BWD_BUFFERS * 3 * sizeof(float) <= 1024, "the workspace's spare bytes must cover the 16-byte rounding");

size_t nerf_b200_march_bwd_workspace_bytes(int64_t N, int S, const NerfNetParams* net) {
  if (check_exact_net(net)) return 0;
  const long long rows = (long long)(N < BWD_RAYS_PER_SLAB ? N : BWD_RAYS_PER_SLAB) * S;
  return (size_t)rows * (3 + bwd_floats_per_row(*net)) * 4 + 1024;
}

static int gemm_nn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, long long M, int N, int K, int beta, cudaStream_t st) {
  dim3 grid(cdiv(M, GT), cdiv(N, GT));
  sgemm_nn_kernel<<<grid, 256, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K, beta);
  NB_LAUNCH_OK("sgemm_nn_kernel");
  return 0;
}
// The two row-reductions below split M over slabs / blocks; with more than one, their partials go to `scratch` (one of the
// pass's [M, W] buffers that is free at the call) and sum_partials_kernel adds them in order.  The partials fit: slabs need
// cdiv(M, 2048) * K1 * N <= M * W floats (K1 <= W, and N <= 1024 <= M / cdiv(M, 2048) when M > 2048); blocks need
// cdiv(M, 256) * C <= M * W floats (C <= W).
static int sum_partials(const float* part, int nparts, int rows, int cols, float* dst, int ld, cudaStream_t st) {
  sum_partials_kernel<<<cdiv((long long)rows * cols, 256), 256, 0, st>>>(part, nparts, rows, cols, dst, ld);
  NB_LAUNCH_OK("sum_partials_kernel");
  return 0;
}
static int gemm_tn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, long long M, int K1, int N, float* scratch,
                   long long scratch_floats, cudaStream_t st) {
  const int slab = 2048;
  const int nslab = cdiv(M, slab);
  float* part = nslab > 1 ? scratch : nullptr;
  NB_CHECK_ARG(nslab == 1 || (long long)nslab * K1 * N <= scratch_floats, "internal: wgrad partials do not fit the scratch buffer");
  dim3 grid(cdiv(K1, GT), cdiv(N, GT), nslab);
  sgemm_tn_kernel<<<grid, 256, 0, st>>>(A, lda, B, ldb, C, ldc, M, K1, N, slab, part);
  NB_LAUNCH_OK("sgemm_tn_kernel");
  return part ? sum_partials(part, nslab, K1, N, C, ldc, st) : 0;
}
// colsum NULL: the ReLU mask alone, no partials (scratch may be NULL)
static int mask_colsum(float* d, int ldd, const float* h, int ldh, long long M, int C, float* colsum, float* scratch,
                       long long scratch_floats, cudaStream_t st) {
  const int rpb = 256;
  const int nblk = cdiv(M, rpb);
  float* part = (nblk > 1 && colsum) ? scratch : nullptr;
  NB_CHECK_ARG(!colsum || nblk == 1 || (long long)nblk * C <= scratch_floats, "internal: column-sum partials do not fit the scratch buffer");
  dim3 grid(nblk, cdiv(C, 64));
  relu_mask_colsum_kernel<<<grid, 64, 0, st>>>(d, ldd, h, ldh, M, C, colsum, rpb, part);
  NB_LAUNCH_OK("relu_mask_colsum_kernel");
  return part ? sum_partials(part, nblk, 1, C, colsum, C, st) : 0;
}
#define NB_TRY(expr) do { if (int rc__ = (expr)) return rc__; } while (0)

static int march_bwd_impl(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                          const NerfRenderCfg* cfg, const NerfOutGrads& g, const NerfNetGrads* grads,
                          void* workspace, size_t workspace_bytes, void* stream) {
  NB_CHECK_ARG(rays && z_vals && net && cfg && grads, "NULL pointer");
  NB_CHECK_ARG(!seeds_none(g), "no output gradient given (every NerfOutGrads member is NULL)");
  if (int rc = check_exact_net(net)) return rc;
  if (N == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int W = net->W, W2 = W / 2, IC = net->input_ch, ICV = net->input_ch_views, D = net->D, rs = cfg->ray_stride;
  NB_CHECK_ARG(workspace && workspace_bytes >= nerf_b200_march_bwd_workspace_bytes(N, S, net), "march_bwd workspace too small");
  for (int64_t n0 = 0; n0 < N; n0 += BWD_RAYS_PER_SLAB) {
    const int64_t nn = (N - n0 < BWD_RAYS_PER_SLAB) ? N - n0 : BWD_RAYS_PER_SLAB;
    const long long M = nn * (long long)S;
    const float* ry = rays + n0 * rs;
    const float* zz = z_vals + n0 * S;
    const float* nz = noise ? noise + n0 * S : nullptr;
    // every one of the BWD_BUFFERS buffers starts on a 16-byte boundary (round4): neither M * (3 + IC + ICV) nor M * W / 2 need
    // be a multiple of 4 (odd M, W = 4k with k odd).  The rounding takes at most BWD_BUFFERS * 12 of the workspace's 1024 spare bytes.
    float* p = static_cast<float*>(workspace);
    float* pts = p;        p += round4(M * 3);
    SimtSave sv;
    sv.enc = p;            p += round4(M * IC);
    sv.encv = p;           p += round4(M * ICV);
    sv.h = p;              p += round4((long long)D * M * W);
    sv.feat = p;           p += round4(M * W);
    sv.hv = p;             p += round4(M * W2);
    float* raw = p;        p += round4(M * 4);
    float* d_raw = p;      p += round4(M * 4);
    float* dh0 = p;        p += round4(M * W);
    float* dh1 = p;        p += round4(M * W);
    float* d_hv = p;       p += round4(M * W2);
    if (!net->use_viewdirs) { sv.encv = nullptr; sv.feat = nullptr; sv.hv = nullptr; }
    // 1. recompute the pass in fp32 with saved activations
    pts_kernel<<<cdiv(M, 256), 256, 0, st>>>(ry, rs, zz, M, S, pts);
    NB_LAUNCH_OK("pts_kernel");
    NB_TRY(launch_mlp_simt(pts, net->use_viewdirs ? ry + 8 : nullptr, rs, M, S, *net, cfg->multires, cfg->multires_views, raw, sv, st));
    // 2. compositing adjoint -> dL/draw
    NB_TRY(raw2outputs_bwd_impl(raw, zz, ry + 3, rs, nz, nn, S, cfg->white_bkgd, seeds_at(g, n0, S), nullptr, d_raw, st));
    const float* h_last = sv.h + (size_t)(D - 1) * M * W;
    const long long sc = M * W;                      // floats of each [M, W] buffer: the partials' scratch is one that is free
    if (net->use_viewdirs) {
      // 3. rgb_linear (run_nerf_helpers.py:114)
      NB_TRY(gemm_tn(d_raw, 4, sv.hv, W2, grads->rgb_w, W2, M, 3, W2, dh0, sc, st));
      NB_TRY(mask_colsum(d_raw, 4, nullptr, 0, M, 3, grads->rgb_b, dh0, sc, st));
      NB_TRY(gemm_nn(d_raw, 4, net->rgb_w, W2, d_hv, W2, M, W2, 3, 0, st));
      // 4. views_linears[0] on cat([feature, input_views]) (:108-112)
      NB_TRY(mask_colsum(d_hv, W2, sv.hv, W2, M, W2, grads->views_b, dh0, sc, st));
      NB_TRY(gemm_tn(d_hv, W2, sv.feat, W, grads->views_w, W + ICV, M, W2, W, dh0, sc, st));
      NB_TRY(gemm_tn(d_hv, W2, sv.encv, ICV, grads->views_w + W, W + ICV, M, W2, ICV, dh0, sc, st));
      NB_TRY(gemm_nn(d_hv, W2, net->views_w, W + ICV, dh0, W, M, W, W2, 0, st));                // d_feature
      // 5. feature_linear and alpha_linear both read the last hidden layer (:106-107)
      NB_TRY(gemm_tn(dh0, W, h_last, W, grads->feature_w, W, M, W, W, dh1, sc, st));
      NB_TRY(mask_colsum(dh0, W, nullptr, 0, M, W, grads->feature_b, dh1, sc, st));
      NB_TRY(gemm_tn(d_raw + 3, 4, h_last, W, grads->alpha_w, W, M, 1, W, dh1, sc, st));
      NB_TRY(mask_colsum(d_raw + 3, 4, nullptr, 0, M, 1, grads->alpha_b, dh1, sc, st));
      NB_TRY(gemm_nn(dh0, W, net->feature_w, W, dh1, W, M, W, W, 0, st));
      NB_TRY(gemm_nn(d_raw + 3, 4, net->alpha_w, W, dh1, W, M, W, 1, 1, st));
    } else {
      // 3'. output_linear (:117): only its first four rows ever reach the loss (run_nerf.py:187 note); rows >= 4 get zero gradient
      NB_TRY(gemm_tn(d_raw, 4, h_last, W, grads->output_w, W, M, 4, W, dh0, sc, st));
      NB_TRY(mask_colsum(d_raw, 4, nullptr, 0, M, 4, grads->output_b, dh0, sc, st));
      NB_TRY(gemm_nn(d_raw, 4, net->output_w, W, dh1, W, M, W, 4, 0, st));
    }
    // 6. pts_linears, last to first (:99-103); skip layer input = cat([input_pts, h])
    float* dcur = dh1;
    float* dnext = dh0;
    for (int l = D - 1; l >= 0; --l) {
      NB_TRY(mask_colsum(dcur, W, sv.h + (size_t)l * M * W, W, M, W, grads->pts_b[l], dnext, sc, st));
      const bool after_skip = (l > 0) && (l - 1 == net->skip);
      const int Kl = (l == 0) ? IC : (after_skip ? W + IC : W);
      if (l == 0) {
        NB_TRY(gemm_tn(dcur, W, sv.enc, IC, grads->pts_w[0], Kl, M, W, IC, dnext, sc, st));
      } else {
        const float* hprev = sv.h + (size_t)(l - 1) * M * W;
        const int off = after_skip ? IC : 0;
        if (after_skip) NB_TRY(gemm_tn(dcur, W, sv.enc, IC, grads->pts_w[l], Kl, M, W, IC, dnext, sc, st));
        NB_TRY(gemm_tn(dcur, W, hprev, W, grads->pts_w[l] + off, Kl, M, W, W, dnext, sc, st));
        NB_TRY(gemm_nn(dcur, W, net->pts_w[l] + off, Kl, dnext, W, M, W, W, 0, st));
        float* t = dcur; dcur = dnext; dnext = t;
      }
    }
  }
  return 0;
}

int nerf_b200_march_bwd(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                        const void* packed, const NerfRenderCfg* cfg, const float* g_rgb, const NerfNetGrads* grads,
                        void* workspace, size_t workspace_bytes, void* stream) {
  (void)packed;
  return march_bwd_impl(rays, z_vals, noise, N, S, net, cfg, rgb_seed(g_rgb), grads, workspace, workspace_bytes, stream);
}

int nerf_b200_march_bwd_outs(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                             const void* packed, const NerfRenderCfg* cfg, const NerfOutGrads* g, const NerfNetGrads* grads,
                             void* workspace, size_t workspace_bytes, void* stream) {
  (void)packed;
  NB_CHECK_ARG(g, "NULL pointer");
  return march_bwd_impl(rays, z_vals, noise, N, S, net, cfg, *g, grads, workspace, workspace_bytes, stream);
}

// ---- the density gradient at arbitrary points (exact path) ----------------------------------------
// Slabs of up to GRAD_SLAB points: mlp_simt_kernel in save mode (enc, h; raw for sigma) with one zero view direction, the seed
// dA_{D-1}, then march_bwd_impl's chain through pts_linears[D-1..1] (gemm_nn, ReLU mask), d_enc = dA_{s+1} W_{s+1}[:, :IC] +
// dA_0 W_0, and the encoding's Jacobian.  Workspace: 256 B (the zero view direction) | enc [slab, IC] | h [D][slab, W] |
// raw [slab, 4] | dA ping/pong 2 x [slab, W] | d_enc [slab, IC], each buffer on a 16-byte boundary (round4), 256 spare bytes.
static const long long GRAD_SLAB = 1ll << 14;
static const int GRAD_BUFFERS = 6;
static_assert(GRAD_BUFFERS * 3 * sizeof(float) <= 256, "the workspace's spare bytes must cover the 16-byte rounding");

size_t nerf_b200_density_gradient_workspace_bytes(int64_t P, const NerfNetParams* net) {
  if (P < 0 || check_exact_net(net)) return 0;
  const long long slab = P < GRAD_SLAB ? P : GRAD_SLAB;
  const size_t per_row = 2 * (size_t)net->input_ch + (size_t)net->D * net->W + 2 * (size_t)net->W + 4;
  return 256 + (size_t)slab * per_row * 4 + 256;
}

int nerf_b200_density_gradient(const float* pts, int64_t P, const NerfNetParams* net, int L, float* sigma, float* grad,
                               void* workspace, size_t workspace_bytes, void* stream) {
  NB_CHECK_ARG(pts && net && sigma && grad && workspace, "NULL pointer");
  NB_CHECK_ARG(P >= 0, "P must be >= 0 (got %lld)", (long long)P);
  if (int rc = check_exact_net(net)) return rc;
  NB_CHECK_ARG(L >= 0 && 3 + 6 * L == net->input_ch, "multires %d does not match input_ch %d", L, net->input_ch);
  const size_t need = nerf_b200_density_gradient_workspace_bytes(P, net);
  NB_CHECK_ARG(workspace_bytes >= need, "workspace too small: need %zu bytes", need);
  NB_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "workspace must start on a 16-byte boundary");
  if (P == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int W = net->W, IC = net->input_ch, D = net->D;
  const long long slab = P < GRAD_SLAB ? P : GRAD_SLAB;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const float* zero_dir = reinterpret_cast<const float*>(ws);
  float* p = reinterpret_cast<float*>(ws + 256);
  SimtSave sv;
  memset(&sv, 0, sizeof(sv));
  sv.enc = p;            p += round4(slab * IC);
  sv.h = p;              p += round4((long long)D * slab * W);
  float* raw = p;        p += round4(slab * 4);
  float* dA0 = p;        p += round4(slab * W);
  float* dA1 = p;        p += round4(slab * W);
  float* d_enc = p;
  const float* w_sigma = net->use_viewdirs ? net->alpha_w : net->output_w + 3 * (size_t)W;
  NB_CUDA(cudaMemsetAsync(ws, 0, 256, st));
  for (long long m0 = 0; m0 < P; m0 += slab) {
    const long long M = P - m0 < slab ? P - m0 : slab;
    const float* x = pts + m0 * 3;
    NB_TRY(launch_mlp_simt(x, zero_dir, 0, M, 1, *net, L, 0, raw, sv, st));
    raw_sigma_kernel<<<cdiv(M, 256), 256, 0, st>>>(raw, M, sigma + m0);
    NB_LAUNCH_OK("raw_sigma_kernel");
    sigma_seed_kernel<<<cdiv(M * W, 256), 256, 0, st>>>(sv.h + (size_t)(D - 1) * M * W, w_sigma, M, W, dA0);
    NB_LAUNCH_OK("sigma_seed_kernel");
    // pts_linears, last to first; the skip layer's input is cat([input_pts, h]): its first IC columns go to d_enc
    float* dcur = dA0;
    float* dnext = dA1;
    for (int l = D - 1; l >= 1; --l) {
      const bool after_skip = l - 1 == net->skip;
      const int Kl = after_skip ? W + IC : W, off = after_skip ? IC : 0;
      if (after_skip) NB_TRY(gemm_nn(dcur, W, net->pts_w[l], Kl, d_enc, IC, M, IC, W, 0, st));
      NB_TRY(gemm_nn(dcur, W, net->pts_w[l] + off, Kl, dnext, W, M, W, W, 0, st));
      NB_TRY(mask_colsum(dnext, W, sv.h + (size_t)(l - 1) * M * W, W, M, W, nullptr, nullptr, 0, st));
      float* t = dcur; dcur = dnext; dnext = t;
    }
    NB_TRY(gemm_nn(dcur, W, net->pts_w[0], IC, d_enc, IC, M, IC, W, net->skip >= 0 ? 1 : 0, st));
    enc_jacobian_kernel<<<cdiv(M, 256), 256, 0, st>>>(d_enc, IC, L, x, M, grad + m0 * 3);
    NB_LAUNCH_OK("enc_jacobian_kernel");
  }
  return 0;
}

// ---- tensor-core backward of one pass (bwd_wg.cuh) ------------------------------------------------
namespace {
struct BwdTcLayout { size_t off_amax, off_draw, off_encv, off_dsum, off_gv, off_partial, off_grad, total; long long part_floats; };
// r[0, n): the dW blocks' reductions (r[i] belongs to w[i]); r[n, nr): the bias sums', alpha_linear's and the seed kernels'
struct BwdTcJobs {
  int n, nr; bool overflow; WgradJob w[WG2_MAX_JOBS]; float* db[WG2_MAX_JOBS]; ReduceJob r[WG2_MAX_REDUCE]; int total_ctas;
  long long part_floats, extra_end;
  void reduce(long long off, long long gstride, int nparts, int Nc, float* dst, int scaled) {   // dst[i] += sum of nparts rows
    ReduceJob& q = r[nr++];
    q.part_off = off; q.gstride = gstride; q.ncta = nparts; q.Mc = 1; q.Nc = Nc; q.n_valid = Nc; q.ldw = Nc; q.dst = dst; q.scaled = scaled;
  }
};

// jobs of the weight gradient (128-row blocks of dW) and their CTA ranges (proportional to the bytes each job streams per tile).
// Every job gets at least one CTA: the caller rejects `sms` < J.n (and J.overflow: more jobs than WG2_MAX_JOBS).
// The dW blocks take the partial region's lower half (at most sms x 128 x 256 floats); the bias sums and alpha_linear's partials
// follow from sms x 128 x 256 up to J.extra_end.
BwdTcJobs make_bwd_jobs(const NerfNetParams& n, const NerfNetGrads* g, int sms) {
  BwdTcJobs J;
  memset(&J, 0, sizeof(J));
  const int D = n.D, W = n.W, IC = n.input_ch;
  auto add = [&](uint32_t a_off, int Mc, uint32_t b_off, int Nc, float* dst, int ldw, int n_valid, float* db) {
    for (int m0 = 0; m0 < Mc; m0 += 128) {
      if (J.n == WG2_MAX_JOBS) { J.overflow = true; return; }
      WgradJob& w = J.w[J.n];
      ReduceJob& r = J.r[J.n];
      w.a_off = a_off; w.a_cols = Mc; w.m0 = m0; w.b_off = b_off; w.Nc = Nc; w.db_off = -1; w.alpha_off = -1;
      J.db[J.n] = db ? db + m0 : nullptr;
      r.Mc = 128; r.Nc = Nc; r.scaled = 1; r.n_valid = n_valid; r.ldw = ldw; r.dst = dst ? dst + (size_t)m0 * ldw : nullptr;
      ++J.n;
    }
  };
  // job 0: G = d_hv^T h_{D-1} (-> views_linears[0].weight[:, :W] through views_feat_wgrad_kernel; its reduce target is a scratch
  // block set by the caller);  jobs 1, 2: feature_linear = d_feat^T h_{D-1} (job 1 also forms alpha_linear's gradient).
  // Without view directions the pts layers are all (output_linear's gradient comes from dA_seed_output_kernel).
  if (n.use_viewdirs) {
    add(0, 128, rec_act_h(D - 1), 256, nullptr, 256, 256, g ? g->views_b : nullptr);
    add(rec_grad_step(0), 256, rec_act_h(D - 1), 256, g ? g->feature_w : nullptr, W, W, g ? g->feature_b : nullptr);
  }
  for (int l = D - 1; l >= 1; --l) {
    const bool sk = (n.skip >= 0 && l == n.skip + 1);
    add(rec_grad_dA(l, D), 256, rec_act_h(l - 1), 256, g ? g->pts_w[l] + (sk ? IC : 0) : nullptr, sk ? W + IC : W, W, g ? g->pts_b[l] : nullptr);
    if (sk) add(rec_grad_dA(l, D), 256, 0, 64, g ? g->pts_w[l] : nullptr, W + IC, IC, nullptr);        // the [input_pts] columns
  }
  add(rec_grad_dA(0, D), 256, 0, 64, g ? g->pts_w[0] : nullptr, IC, IC, g ? g->pts_b[0] : nullptr);
  // CTAs per job ~ the bytes it streams per tile (128 + Nc columns)
  auto cost = [&](int i) { return (double)(128 + J.w[i].Nc); };
  if (J.overflow || J.n > sms) return J;
  double tot = 0;
  for (int i = 0; i < J.n; ++i) tot += cost(i);
  int used = 0;
  double frac[WG2_MAX_JOBS];
  for (int i = 0; i < J.n; ++i) {
    const double x = (double)sms * cost(i) / tot;
    int c = (int)x;
    if (c < 1) c = 1;
    frac[i] = x - c;
    J.w[i].ncta = c;
    used += c;
  }
  while (used < sms) {                               // leftovers: largest remainder first
    int b = 0;
    for (int i = 1; i < J.n; ++i) if (frac[i] > frac[b]) b = i;
    ++J.w[b].ncta; ++used; frac[b] -= 1.0;
  }
  while (used > sms) {                               // (rounding up to one CTA per job overshot: take from the largest)
    int b = 0;
    for (int i = 1; i < J.n; ++i) if (J.w[i].ncta > J.w[b].ncta) b = i;
    --J.w[b].ncta; --used;
  }
  int cta = 0;
  long long pf = 0;
  for (int i = 0; i < J.n; ++i) {
    J.w[i].cta0 = cta; cta += J.w[i].ncta;
    J.w[i].part_off = pf; J.r[i].part_off = pf; J.r[i].gstride = 128LL * J.w[i].Nc; J.r[i].ncta = J.w[i].ncta;
    pf += (long long)J.w[i].ncta * 128 * J.w[i].Nc;
  }
  J.total_ctas = cta; J.part_floats = pf;
  J.nr = J.n;
  long long xf = (long long)sms * 128 * 256;
  for (int i = 0; i < J.n; ++i) {
    if (!J.db[i]) continue;
    J.w[i].db_off = xf;                              // [ncta][4 warp quarters][128]
    J.reduce(xf, 128, 4 * J.w[i].ncta, 128, J.db[i], 1);
    xf += 512LL * J.w[i].ncta;
  }
  if (n.use_viewdirs && g) {                         // feature job, first block: alpha_linear
    const int G = J.w[1].ncta;
    J.w[1].alpha_off = xf;                           // [G][2 row halves][256] weight, then [G][2] bias
    J.reduce(xf, 256, 2 * G, 256, g->alpha_w, 0);
    J.reduce(xf + 512LL * G, 1, 2 * G, 1, g->alpha_b, 0);
    xf += 514LL * G;
  }
  J.extra_end = xf;
  return J;
}

// split: the gradient records are the split backward's hi + lo pairs
BwdTcLayout make_bwd_layout(long long N, int S, const NerfNetParams& n, const TilePlan& plan, long long part_floats, bool split = false) {
  BwdTcLayout L;
  auto up = [](size_t x) { return (x + 1023) & ~(size_t)1023; };
  size_t o = 0;
  L.off_amax = o;    o = up(o + 256);
  L.off_draw = o;    o = up(o + (size_t)N * S * 16);
  L.off_encv = o;    o = up(o + (size_t)N * (n.input_ch_views > 0 ? n.input_ch_views : 1) * 4);
  L.off_dsum = o;    o = up(o + (size_t)N * 128 * 4);
  L.off_gv = o;      o = up(o + (size_t)(128 * 256 + 128) * 4);      // G = d_hv^T h_{D-1} (reduced) and this pass's db_v
  L.off_partial = o; o = up(o + (size_t)part_floats * 4);
  L.off_grad = o;    o = up(o + (size_t)plan.n_tiles * rec_grad_bytes(n.D) * (split ? 2 : 1));
  L.total = o; L.part_floats = part_floats;
  return L;
}
}  // namespace

static size_t bwd_pass_bytes(int64_t N, int S, const NerfNetParams* net, bool split = false) {
  const int sms = num_sms();
  const TilePlan plan = make_tile_plan(N, S, sms);
  return make_bwd_layout(N, S, *net, plan, (long long)sms * 256 * 256, split).total + 1024;
}

size_t nerf_b200_march_bwd_tc_workspace_bytes(int64_t N, int S, const NerfNetParams* net) {
  if (!net || check_tc_net(net) || N <= 0 || S <= 0) return 0;
  return bwd_pass_bytes(N, S, net);
}

// introspection for tests and tools: where nerf_b200_march_bwd_tc keeps its intermediates inside the (1 KB-aligned)
// workspace and how the tiles are laid out.  out[0..11] = off_d_raw, off_grad_records, rec_act_bytes, rec_mask_bytes,
// rec_grad_bytes, grid, rays_per_cta, nst, n_tiles, off_amax, off_dsum, off_partial
static int bwd_layout(int64_t N, int S, const NerfNetParams* net, int64_t* out, bool split) {
  if (int rc = check_tc_net(net)) return rc;
  NB_CHECK_ARG(out && N > 0 && S > 0, "bad arguments");
  const int sms = num_sms();
  const TilePlan plan = make_tile_plan(N, S, sms);
  const BwdTcLayout LY = make_bwd_layout(N, S, *net, plan, (long long)sms * 256 * 256, split);
  const int64_t m = split ? 2 : 1;
  out[0] = (int64_t)LY.off_draw; out[1] = (int64_t)LY.off_grad; out[2] = m * rec_act_bytes(net->D); out[3] = rec_mask_bytes(net->D);
  out[4] = m * rec_grad_bytes(net->D); out[5] = plan.grid; out[6] = plan.rays_per_cta; out[7] = plan.nst; out[8] = plan.n_tiles;
  out[9] = (int64_t)LY.off_amax; out[10] = (int64_t)LY.off_dsum; out[11] = (int64_t)LY.off_partial;
  return 0;
}

int nerf_b200_march_bwd_tc_layout(int64_t N, int S, const NerfNetParams* net, int64_t* out) { return bwd_layout(N, S, net, out, false); }
// the same for the split backward: out[2] and out[4] are the strides of the hi + lo record pairs (the lo record follows the hi one)
int nerf_b200_march_bwd_split_layout(int64_t N, int S, const NerfNetParams* net, int64_t* out) { return bwd_layout(N, S, net, out, true); }

namespace {
// One pass of the tensor-core backward, in its phases: prologue (loss scale, compositing adjoint, seed tiles), dgrad chain,
// weight gradients, view-column gradients.
struct BwdTcPass {
  const float* rays; const float* z; const float* noise; int64_t N; int S; const NerfNetParams* net; const void* packed;
  const NerfRenderCfg* cfg; const float* raw; const NerfTrainSave* save; NerfOutGrads seeds; const NerfNetGrads* grads;
  DeviceState* ds; TilePlan plan; BwdTcLayout LY; PackLayout PL; BwdTcJobs J;
  unsigned int* amax; float *d_raw, *encv, *dsum, *gv, *dbv, *partial; uint8_t* grec; const uint8_t *act, *mask;
  int seed_grid; long long seed_off, views_rays;      // seed kernels: blocks, partial rows from `seed_off`; rays per views block
  bool split;                                         // the split backward (precision TC_SPLIT, split records and image)
  uint32_t ract, rgrad;                               // per-tile strides of the activation and gradient records

  // the refusals of a pass, before anything is launched
  int check() const {
    NB_CHECK_ARG(rays && z && net && packed && cfg && raw && save && grads, "NULL pointer");
    if (split) NB_CHECK_ARG(cfg->precision == NERF_B200_PREC_TC_SPLIT, "the split backward needs precision TC_SPLIT");
    else NB_CHECK_ARG(cfg->precision != NERF_B200_PREC_TC_SPLIT, NB_SPLIT_TRAIN_MSG);
    NB_CHECK_ARG(!seeds_none(seeds), "no output gradient given for a backward pass (g_rgb / every NerfOutGrads member is NULL)");
    if (int rc = check_tc_net(net)) return rc;
    NB_CHECK_ARG(net->use_viewdirs || net->output_ch >= 4, "output_linear needs output_ch >= 4 (got %d)", net->output_ch);
    NB_CHECK_ARG(S > 0, "S must be positive");
    return 0;
  }

  int run(void* workspace, size_t workspace_bytes, cudaStream_t st) {
    NB_TRY(init(workspace, workspace_bytes));
    NB_TRY(prologue(st));
    NB_TRY(dgrad(st));
    NB_TRY(wgrad(st));
    return heads(st);
  }

  int init(void* workspace, size_t workspace_bytes) {
    ds = device_state();
    plan = make_tile_plan(N, S, ds->sms);
    LY = make_bwd_layout(N, S, *net, plan, (long long)ds->sms * 256 * 256, split);
    ract = rec_act_bytes(net->D) * (split ? 2u : 1u);
    rgrad = rec_grad_bytes(net->D) * (split ? 2u : 1u);
    uint8_t* ws = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~(uintptr_t)1023);
    NB_CHECK_ARG(workspace && workspace_bytes >= LY.total + (size_t)(ws - static_cast<uint8_t*>(workspace)), "march_bwd_tc workspace too small (%zu < %zu)", workspace_bytes, LY.total + 1024);
    NB_CHECK_ARG(save->act && save->mask && save->act_bytes >= (size_t)plan.n_tiles * ract && save->mask_bytes >= (size_t)plan.n_tiles * rec_mask_bytes(net->D),
                 "training-mode records missing or too small");
    PL = split ? make_pack_layout_split_train(*net) : make_pack_layout(*net);
    amax = reinterpret_cast<unsigned int*>(ws + LY.off_amax);
    d_raw = reinterpret_cast<float*>(ws + LY.off_draw);
    encv = reinterpret_cast<float*>(ws + LY.off_encv);
    dsum = reinterpret_cast<float*>(ws + LY.off_dsum);
    gv = reinterpret_cast<float*>(ws + LY.off_gv);
    dbv = gv + 128 * 256;
    partial = reinterpret_cast<float*>(ws + LY.off_partial);
    grec = ws + LY.off_grad;
    act = static_cast<const uint8_t*>(save->act);
    mask = static_cast<const uint8_t*>(save->mask);
    // every partial sum lives in the partial region (sms x 256 x 256 floats): the dW blocks in its lower half, above them the bias
    // and alpha_linear partials, then the seed kernels' rows; the views kernel's rows reuse the upper half once those are reduced
    const int sms = ds->sms;
    J = make_bwd_jobs(*net, grads, sms);
    NB_CHECK_ARG(!J.overflow && J.n <= sms, "weight gradient: %d jobs need at least as many CTAs (have %d; at most %d jobs)", J.n, sms, WG2_MAX_JOBS);
    const long long cap = (long long)sms * 256 * 256, upper = (long long)sms * 128 * 256;
    seed_grid = (int)(plan.n_tiles < (net->use_viewdirs ? 3 : 2) * sms ? plan.n_tiles : (net->use_viewdirs ? 3 : 2) * sms);
    seed_off = J.extra_end;
    const long long seed_floats = (long long)seed_grid * (net->use_viewdirs ? SEED_HEADS_PART : SEED_OUT_PART);
    views_rays = (N + sms - 1) / sms;
    const long long views_floats = net->use_viewdirs ? (long long)sms * (net->input_ch_views + 1) * 128 : 0;
    NB_CHECK_ARG(J.part_floats <= upper && seed_off + seed_floats <= cap && upper + views_floats <= cap,
                 "internal: backward partials exceed the partial region");
    if (split) NB_TRY(smem_optin_once((const void*)dgrad_split_kernel, DS_ALLOC));
    else NB_TRY(smem_optin_once((const void*)dgrad_wg_kernel, SM_ALLOC));
    NB_TRY(smem_optin_once((const void*)wgrad_wg_kernel, WG2_TOTAL));
    return 0;
  }

  // 1. compositing adjoint -> dL/draw (SURVEY App. E) and the loss scale: from max |dL/drgb_map| (absmax_kernel) when rgb_map
  // is the only seed, else from the adjoint's max over all effective seeds;  2. seed of the chain: d_hv tiles, or
  // without view directions dA_{D-1} tiles (+ output_linear's gradient).  Both read amax after the adjoint, on the same stream.
  int prologue(cudaStream_t st) {
    const int D = net->D;
    NB_CUDA(cudaMemsetAsync(amax, 0, 256, st));
    if (net->use_viewdirs) NB_CUDA(cudaMemsetAsync(gv, 0, (size_t)(128 * 256 + 128) * 4, st));
    if (seeds_rgb_only(seeds)) {
      absmax_kernel<<<cdiv(N * 3, 1024) < 64 ? cdiv(N * 3, 1024) : 64, 256, 0, st>>>(seeds.rgb_map, N * 3, amax);
      NB_LAUNCH_OK("absmax_kernel");
      NB_TRY(raw2outputs_bwd_impl(raw, z, rays + 3, cfg->ray_stride, noise, N, S, cfg->white_bkgd, seeds, nullptr, d_raw, st));
    } else {
      NB_TRY(raw2outputs_bwd_impl(raw, z, rays + 3, cfg->ray_stride, noise, N, S, cfg->white_bkgd, seeds, amax, d_raw, st));
    }
    if (!net->use_viewdirs) {
      SeedOutParams so;
      so.d_raw = d_raw; so.mask = mask; so.act = act; so.grad = grec; so.out_w = net->output_w; so.amax = amax;
      so.N = N; so.S = S; so.rays_per_cta = plan.rays_per_cta; so.nst_plan = plan.nst; so.D = D;
      so.rec_mask = rec_mask_bytes(D); so.rec_act = ract; so.rec_grad = rgrad; so.n_tiles = plan.n_tiles;
      so.part = partial + seed_off;
      if (split) dA_seed_output_split_kernel<<<seed_grid, 256, 0, st>>>(so);
      else dA_seed_output_kernel<<<seed_grid, 256, 0, st>>>(so);
      NB_LAUNCH_OK(split ? "dA_seed_output_split_kernel" : "dA_seed_output_kernel");
      J.reduce(seed_off, SEED_OUT_PART, seed_grid, 1024, grads->output_w, 0);
      J.reduce(seed_off + 1024, SEED_OUT_PART, seed_grid, 4, grads->output_b, 0);
      return 0;
    }
    SeedParams sp;
    sp.d_raw = d_raw; sp.mask = mask; sp.act = act; sp.grad = grec; sp.rgb_w = net->rgb_w; sp.amax = amax;
    sp.N = N; sp.S = S; sp.rays_per_cta = plan.rays_per_cta; sp.nst_plan = plan.nst; sp.D = D;
    sp.rec_mask = rec_mask_bytes(D); sp.rec_act = ract; sp.rec_grad = rgrad; sp.n_tiles = plan.n_tiles;
    sp.part = partial + seed_off;
    if (split) dhv_seed_heads_split_kernel<<<seed_grid, 256, 0, st>>>(sp);
    else dhv_seed_heads_kernel<<<seed_grid, 256, 0, st>>>(sp);
    NB_LAUNCH_OK(split ? "dhv_seed_heads_split_kernel" : "dhv_seed_heads_kernel");
    J.reduce(seed_off, SEED_HEADS_PART, seed_grid, 384, grads->rgb_w, 0);
    J.reduce(seed_off + 384, SEED_HEADS_PART, seed_grid, 3, grads->rgb_b, 0);
    return 0;
  }

  // 3. dgrad chain, one CTA per forward CTA (the forward's tile order)
  int dgrad(cudaStream_t st) {
    const int D = net->D;
    const uint8_t* pk = static_cast<const uint8_t*>(packed);
    DgradParams dp;
    const bool views = net->use_viewdirs != 0;
    dp.mask = mask; dp.grad = grec; dp.amax = amax;
    dp.d_raw = views ? d_raw : nullptr; dp.alpha_w = views ? net->alpha_w : nullptr;
    dp.chunks = pk + PL.off_bwd;
    dp.N = N; dp.S = S; dp.rays_per_cta = plan.rays_per_cta; dp.nst_plan = plan.nst; dp.D = D;
    dp.rec_mask = rec_mask_bytes(D); dp.rec_grad = rgrad;
    dp.vc0 = 0; dp.vc1 = plan.grid;                   // every CTA of the plan
    dp.first_step = bwd_first_step(net->use_viewdirs);
    // MACs per row of the steps the kernel runs: K = W/2 (step 0) + D steps of W x W, or without view directions D - 1 steps
    const double macs = views ? (double)(net->W / 2) * net->W + (double)D * net->W * net->W : (double)(D - 1) * net->W * net->W;
    TimedLaunch* tl = timing_begin(1, 2.0 * macs * (double)(N * (long long)S), st);
    if (split) dgrad_split_kernel<<<plan.grid, TC_THREADS, DS_ALLOC, st>>>(dp, reinterpret_cast<const float*>(pk + PL.off_wscale));
    else dgrad_wg_kernel<<<plan.grid, TC_THREADS, SM_ALLOC, st>>>(dp);
    timing_end(tl, st);
    NB_LAUNCH_OK(split ? "dgrad_split_kernel" : "dgrad_wg_kernel");
    return 0;
  }

  // 4. weight gradients (layer-major) + bias gradients on all SMs, then the reduction of the per-CTA partials (and of the seed
  // kernels' partial rows) in CTA order (adds into the gradient tensors).  Split: dW = dA_hi^T H_hi + dA_lo^T H_hi + dA_hi^T H_lo
  // as three launches of the same kernel on the hi and lo records, each reduced (added into the tensors) before the next
  // reuses the partial region; the bias sums take dA_hi then dA_lo, alpha_linear's weight H_hi then H_lo (its bias, the sum of
  // d_sigma, once: from the first launch).
  int wgrad(cudaStream_t st) {
    if (!split) return wgrad_launch(act, grec, 0, J.nr, true, true, st);
    const int nd = J.n, ndb = [&] { int k = 0; for (int i = 0; i < J.n; ++i) k += J.w[i].db_off >= 0; return k; }();
    const int na = (net->use_viewdirs && grads) ? 1 : 0;             // alpha_linear.weight's reduction (its bias's follows it)
    NB_TRY(wgrad_launch(act, grec, 0, J.nr, true, true, st));                                               // hi, hi (+ seed heads)
    NB_TRY(wgrad_launch(act, grec + rec_grad_split_lo(net->D), nd, nd + ndb, true, false, st));              // lo dA, hi H
    return wgrad_launch(act + rec_split_lo(net->D), grec, nd + ndb, nd + ndb + na, false, true, st);        // hi dA, lo H
  }

  // one weight-gradient launch on the records at a / g and its reduction: the dW jobs, then J.r[r0, r1) (every reduction when
  // r1 = J.nr); `db` / `alpha`: the launch forms the bias sums / alpha_linear's partials
  int wgrad_launch(const uint8_t* a, const uint8_t* g, int r0, int r1, bool db, bool alpha, cudaStream_t st) {
    const int D = net->D;
    const bool views = net->use_viewdirs != 0;
    WgradParams wp;
    memset(&wp, 0, sizeof(wp));
    wp.act = a; wp.grad = g; wp.rec_act = ract; wp.rec_grad = rgrad;
    wp.N = N; wp.S = S; wp.rays_per_cta = plan.rays_per_cta; wp.nst_plan = plan.nst; wp.n_tiles = plan.n_tiles;
    wp.t0 = 0; wp.t1 = (long long)plan.grid * plan.nst * 2;   // every tile of the plan
    wp.partial = partial; wp.d_raw = d_raw; wp.njobs = J.n;
    for (int i = 0; i < J.n; ++i) {
      wp.jobs[i] = J.w[i];
      if (!db) wp.jobs[i].db_off = -1;
      if (!alpha) wp.jobs[i].alpha_off = -1;
    }
    // every Linear but the heads (alpha / rgb_linear and the view columns, or output_linear: other kernels form those)
    const double heads = views ? (double)net->W + 3.0 * (net->W / 2) + (double)net->input_ch_views * (net->W / 2) : (double)net->W * net->output_ch;
    const bool first = a == act && g == grec;         // the algorithmic work is counted once per pass
    TimedLaunch* tl = timing_begin(2, first ? 2.0 * (net_macs_per_row(*net) - heads) * (double)(N * (long long)S) : 0.0, st);
    wgrad_wg_kernel<<<J.total_ctas, WG2_THREADS, WG2_TOTAL, st>>>(wp);
    timing_end(tl, st);
    NB_LAUNCH_OK(split ? "wgrad_wg_kernel (split record pair)" : "wgrad_wg_kernel");
    ReduceParams rp;
    memset(&rp, 0, sizeof(rp));
    if (views) J.r[0].dst = gv;                       // job 0 reduces into the scratch block G
    rp.partial = partial; rp.amax = amax; rp.njobs = 0;
    for (int i = 0; i < J.nr; ++i)
      if (i < J.n || (i >= r0 && i < r1)) rp.jobs[rp.njobs++] = J.r[i];
    dim3 rg(128, rp.njobs);
    wgrad_reduce_kernel<<<rg, 256, 0, st>>>(rp);
    NB_LAUNCH_OK("wgrad_reduce_kernel");
    return 0;
  }

  // 5. the view columns of views_linears[0] (after ALL of the pass's weight-gradient launches); nothing without view directions
  int heads(cudaStream_t st) {
    if (!net->use_viewdirs) return 0;
    const int ICV = net->input_ch_views;
    encv_kernel<<<cdiv(N * ICV, 256), 256, 0, st>>>(rays + 8, cfg->ray_stride, N, ICV, encv);
    NB_LAUNCH_OK("encv_kernel");
    if (split) dhv_ray_sum_split_kernel<<<cdiv(N, 8), 256, 0, st>>>(grec, rgrad, rec_grad_split_lo(net->D), N, S, plan.rays_per_cta, plan.nst, amax, dsum);
    else dhv_ray_sum_kernel<<<cdiv(N, 8), 256, 0, st>>>(grec, rgrad, N, S, plan.rays_per_cta, plan.nst, amax, dsum);
    NB_LAUNCH_OK(split ? "dhv_ray_sum_split_kernel" : "dhv_ray_sum_kernel");
    const int sms = ds->sms;
    const long long voff = (long long)sms * 128 * 256;  // the upper half of the partial region: reduced already (stream order)
    dim3 vg(ICV + 1, sms);
    views_enc_wgrad_kernel<<<vg, 128, 0, st>>>(dsum, encv, N, ICV, views_rays, partial + voff);
    NB_LAUNCH_OK("views_enc_wgrad_kernel");
    ReduceParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.partial = partial; rp.amax = amax; rp.njobs = 2;
    const long long vrow = (long long)(ICV + 1) * 128;
    rp.jobs[0] = ReduceJob{voff, vrow, sms, 128, ICV, ICV, net->W + ICV, 0, grads->views_w + net->W};   // [c][e] -> weight[c][W + e]
    rp.jobs[1] = ReduceJob{voff + (long long)ICV * 128, vrow, sms, 1, 128, 128, 128, 0, dbv};
    wgrad_reduce_kernel<<<dim3(cdiv(128 * ICV, 256), 2), 256, 0, st>>>(rp);
    NB_LAUNCH_OK("wgrad_reduce_kernel");
    views_feat_wgrad_kernel<<<128, 256, 0, st>>>(gv, dbv, net->feature_w, net->feature_b, grads->views_w, net->W + ICV);
    NB_LAUNCH_OK("views_feat_wgrad_kernel");
    return 0;
  }
};

// pass q of a render_rays backward (a zero pass, which check() refuses, when q is NULL); its seeds are `g` when given, else
// {rgb_map = q->g_rgb}
BwdTcPass bind_pass(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfBwdPass* q, const NerfOutGrads* g, bool split) {
  BwdTcPass b;
  memset(&b, 0, sizeof(b));
  b.split = split;
  if (!q) return b;
  b.rays = rays; b.z = q->z_vals; b.noise = q->noise; b.N = N; b.S = q->S; b.net = q->net; b.packed = q->packed; b.cfg = cfg;
  b.raw = q->raw; b.save = q->save; b.seeds = g ? *g : rgb_seed(q->g_rgb); b.grads = q->grads;
  return b;
}

int march_bwd_tc_impl(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                      const void* packed, const NerfRenderCfg* cfg, const float* raw, const NerfTrainSave* save,
                      const NerfOutGrads& g, const NerfNetGrads* grads, void* workspace, size_t workspace_bytes, void* stream,
                      bool split = false) {
  BwdTcPass b;
  memset(&b, 0, sizeof(b));
  b.split = split;
  b.rays = rays; b.z = z_vals; b.noise = noise; b.N = N; b.S = S; b.net = net; b.packed = packed; b.cfg = cfg;
  b.raw = raw; b.save = save; b.seeds = g; b.grads = grads;
  NB_TRY(b.check());
  if (N == 0) return 0;
  return b.run(workspace, workspace_bytes, (cudaStream_t)stream);
}
}  // namespace

int nerf_b200_march_bwd_tc(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                           const void* packed, const NerfRenderCfg* cfg, const float* raw, const NerfTrainSave* save,
                           const float* g_rgb, const NerfNetGrads* grads, void* workspace, size_t workspace_bytes, void* stream) {
  return march_bwd_tc_impl(rays, z_vals, noise, N, S, net, packed, cfg, raw, save, rgb_seed(g_rgb), grads, workspace, workspace_bytes, stream);
}

int nerf_b200_march_bwd_tc_outs(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                                const void* packed, const NerfRenderCfg* cfg, const float* raw, const NerfTrainSave* save,
                                const NerfOutGrads* g, const NerfNetGrads* grads, void* workspace, size_t workspace_bytes, void* stream) {
  NB_CHECK_ARG(g, "NULL pointer");
  return march_bwd_tc_impl(rays, z_vals, noise, N, S, net, packed, cfg, raw, save, *g, grads, workspace, workspace_bytes, stream);
}

// the split backward of one pass (precision TC_SPLIT): the split records of nerf_b200_march_train_split, the split training
// image (nerf_b200_pack_weights_split_train); seeds as nerf_b200_march_bwd_tc_outs
size_t nerf_b200_march_bwd_split_workspace_bytes(int64_t N, int S, const NerfNetParams* net) {
  if (!net || check_tc_net(net) || N <= 0 || S <= 0) return 0;
  return bwd_pass_bytes(N, S, net, true);
}

int nerf_b200_march_bwd_split(const float* rays, const float* z_vals, const float* noise, int64_t N, int S, const NerfNetParams* net,
                              const void* packed, const NerfRenderCfg* cfg, const float* raw, const NerfTrainSave* save,
                              const NerfOutGrads* g, const NerfNetGrads* grads, void* workspace, size_t workspace_bytes, void* stream) {
  NB_CHECK_ARG(g, "NULL pointer");
  return march_bwd_tc_impl(rays, z_vals, noise, N, S, net, packed, cfg, raw, save, *g, grads, workspace, workspace_bytes, stream, true);
}

static size_t render_rays_bwd_bytes(int64_t N, int S_coarse, const NerfNetParams* net_coarse, int S_fine, const NerfNetParams* net_fine, bool split) {
  if (!net_coarse || check_tc_net(net_coarse) || N <= 0 || S_coarse <= 0) return 0;
  size_t b = bwd_pass_bytes(N, S_coarse, net_coarse, split);
  if (net_fine && S_fine > 0) {
    if (check_tc_net(net_fine) || net_fine->use_viewdirs != net_coarse->use_viewdirs) return 0;
    b += bwd_pass_bytes(N, S_fine, net_fine, split);
  }
  return b;
}
size_t nerf_b200_render_rays_bwd_tc_workspace_bytes(int64_t N, int S_coarse, const NerfNetParams* net_coarse, int S_fine, const NerfNetParams* net_fine) {
  return render_rays_bwd_bytes(N, S_coarse, net_coarse, S_fine, net_fine, false);
}
size_t nerf_b200_render_rays_bwd_split_workspace_bytes(int64_t N, int S_coarse, const NerfNetParams* net_coarse, int S_fine, const NerfNetParams* net_fine) {
  return render_rays_bwd_bytes(N, S_coarse, net_coarse, S_fine, net_fine, true);
}

// Backward of both passes of render_rays (run_nerf.py:765-772: loss = img2mse(rgb) + img2mse(rgb0); z_samples is detached, :394,
// so the passes are independent): one pass after the other on `stream`.  The weight-gradient kernel holds a whole SM (384 threads
// x 168 registers), so nothing of the other pass could run beside it.
static int render_rays_bwd_tc_impl(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfBwdPass* coarse, const NerfBwdPass* fine,
                                   const NerfOutGrads* coarse_g, const NerfOutGrads* fine_g, void* workspace, size_t workspace_bytes,
                                   void* stream, bool split = false) {
  BwdTcPass c = bind_pass(rays, N, cfg, coarse, coarse_g, split), f = bind_pass(rays, N, cfg, fine, fine_g, split);
  NB_TRY(c.check());
  if (fine) NB_TRY(f.check());
  NB_CHECK_ARG(!fine || (fine->net->use_viewdirs != 0) == (coarse->net->use_viewdirs != 0),
               "coarse and fine networks must agree on use_viewdirs (they share one ray batch)");
  if (N == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t cb = bwd_pass_bytes(N, coarse->S, coarse->net, split);
  NB_CHECK_ARG(workspace && workspace_bytes >= cb, "render_rays_bwd_tc workspace too small");
  NB_TRY(c.run(workspace, cb, st));
  return fine ? f.run(static_cast<uint8_t*>(workspace) + cb, workspace_bytes - cb, st) : 0;
}

int nerf_b200_render_rays_bwd_tc(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfBwdPass* coarse, const NerfBwdPass* fine,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  return render_rays_bwd_tc_impl(rays, N, cfg, coarse, fine, nullptr, nullptr, workspace, workspace_bytes, stream);
}

int nerf_b200_render_rays_bwd_tc_outs(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfBwdPass* coarse, const NerfBwdPass* fine,
                                      const NerfOutGrads* coarse_g, const NerfOutGrads* fine_g, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  return render_rays_bwd_tc_impl(rays, N, cfg, coarse, fine, coarse_g, fine_g, workspace, workspace_bytes, stream);
}

// the split backward of both passes on one stream (graph-capturable); seeds per pass as NerfOutGrads (rgb_map alone for an rgb loss)
int nerf_b200_render_rays_bwd_split(const float* rays, int64_t N, const NerfRenderCfg* cfg, const NerfBwdPass* coarse, const NerfBwdPass* fine,
                                    const NerfOutGrads* coarse_g, const NerfOutGrads* fine_g, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  NB_CHECK_ARG(coarse_g && (!fine || fine_g), "NULL output gradients");
  return render_rays_bwd_tc_impl(rays, N, cfg, coarse, fine, coarse_g, fine_g, workspace, workspace_bytes, stream, true);
}

// ---- the two ends of the optimisation step (train_step.cuh) ------------------------------------------
int nerf_b200_mse_seed(const float* rgb, const float* target, int64_t N, float grad_scale, float* g_rgb, float* loss_accum, void* stream) {
  NB_CHECK_ARG(rgb && target && g_rgb && loss_accum, "NULL pointer");
  if (N == 0) return 0;
  const long long n3 = N * 3;
  mse_seed_kernel<<<1, MSE_THREADS, 0, (cudaStream_t)stream>>>(rgb, target, n3, 1.0f / (float)n3, grad_scale, g_rgb, loss_accum);
  NB_LAUNCH_OK("mse_seed_kernel");
  return 0;
}

int nerf_b200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float* state,
                        float lr0, float decay_rate, float decay_steps, float beta1, float beta2, float eps, float grad_mul, void* stream) {
  NB_CHECK_ARG(params && grads && exp_avg && exp_avg_sq && state, "NULL pointer");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = cdiv(n, 1024) < 4 * num_sms() ? cdiv(n, 1024) : 4 * num_sms();
  adam_flat_kernel<<<grid, 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, n, state, lr0, decay_rate, decay_steps, beta1, beta2, eps, grad_mul);
  NB_LAUNCH_OK("adam_flat_kernel");
  adam_advance_kernel<<<1, 1, 0, st>>>(state, lr0, decay_rate, decay_steps);
  NB_LAUNCH_OK("adam_advance_kernel");
  return 0;
}

#ifdef NERF_B200_PHASE_PROBE
// Experiments build only (tools/forward_phase_probe.py): zero the forward's phase counters (fused_wg.cuh: Phases) and the
// launch count that picks their slot; copy them out as uint64 [PH_SLOTS][PH_MAX_CTAS][2][PH_N].
int nerf_b200_phase_probe_reset(void) {
  static unsigned long long zeros[PH_SLOTS][PH_MAX_CTAS][2][PH_N];
  NB_CUDA(cudaDeviceSynchronize());
  NB_CUDA(cudaMemcpyToSymbol(g_fwd_phase, zeros, sizeof(zeros)));
  g_phase_launches = 0;
  return 0;
}
int nerf_b200_phase_probe_read(void* out, size_t bytes) {
  NB_CHECK_ARG(out && bytes == sizeof(g_fwd_phase), "out must hold the whole counter table");
  NB_CUDA(cudaDeviceSynchronize());
  NB_CUDA(cudaMemcpyFromSymbol(out, g_fwd_phase, bytes));
  return 0;
}
int nerf_b200_phase_probe_shape(int* slots, int* max_ctas, int* phases) {
  *slots = PH_SLOTS; *max_ctas = PH_MAX_CTAS; *phases = PH_N;
  return 0;
}
#endif

}  // extern "C"
