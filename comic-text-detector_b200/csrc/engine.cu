// libctd_b200.so: C-ABI engine (see include/ctd_b200.h).  Owns device buffers, the weight blob,
// per-shape launch plans (tensor maps) and the optional CUDA graph; runs the op list emitted by
// the Python host "compiler".  No CPU fallback: every entry point fails without an sm_90 GPU.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cstdlib>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "engine.h"

using namespace ctd;

namespace {
thread_local std::string g_create_error;
}  // namespace

int ctd_fail(ctd_handle* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  else g_create_error = buf;
  return code;
}

#define CK(expr)                                                                                      \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) return ctd_fail(h, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

int rows_per_image(int ph, int pw) { return 3 * ((ph / 8) * (pw / 8) + (ph / 16) * (pw / 16) + (ph / 32) * (pw / 32)); }
// op kinds that are one implicit GEMM over packed weights (conv_tc_kernel or conv_simt_kernel)
static bool is_gemm(int kind) { return kind == CTD_OP_CONV || kind == CTD_OP_DECONV4 || kind == CTD_OP_DETECT; }

extern "C" const char* ctd_last_error(const ctd_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

extern "C" void ctd_destroy(ctd_handle* h) {
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  ctd_pipeline_shutdown(h);
  if (h->ev_pre) {   // ctd_preprocess_pages' buffers: free once its last call's kernels ran
    cudaEventSynchronize(h->ev_pre);
    cudaEventDestroy(h->ev_pre);
  }
  cudaFree(h->pre_in);
  cudaFree(h->d_pre_tab);
  for (auto& kv : h->plans)
    if (kv.second.graph) cudaGraphExecDestroy(kv.second.graph);
  for (void* p : h->d_buf) cudaFree(p);
  for (void* p : h->d_buf16) cudaFree(p);
  cudaFree(h->d_wsplit);
  cudaFree(h->d_blob); cudaFree(h->d_pages); cudaFree(h->d_blks); cudaFree(h->d_mask); cudaFree(h->d_mask_u8);
  cudaFree(h->d_lines); cudaFree(h->d_bitmap); cudaFree(h->d_labels);
  cudaFree(h->d_ccl_scratch); cudaFree(h->d_nms_ws); cudaFree(h->d_segrep_scratch); cudaFree(h->d_segrep_rows);
  h->refine_scratch.release(); h->cc_scratch.release(); h->io_scratch.release(); h->in_stage.release();
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->tev0) cudaEventDestroy(h->tev0);
  if (h->tev1) cudaEventDestroy(h->tev1);
  for (auto e : h->op_events) cudaEventDestroy(e);
  for (Slot& s : h->slot) s.release();
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  if (h->ev_fork2) cudaEventDestroy(h->ev_fork2);
  if (h->ev_xjoin) cudaEventDestroy(h->ev_xjoin);
  if (h->ev_join2) cudaEventDestroy(h->ev_join2);
  if (h->ev_tin) cudaEventDestroy(h->ev_tin);
  if (h->ev_tout) cudaEventDestroy(h->ev_tout);
  if (h->side) cudaStreamDestroy(h->side);
  if (h->side2) cudaStreamDestroy(h->side2);
  if (h->copy_in) cudaStreamDestroy(h->copy_in);
  if (h->copy_out) cudaStreamDestroy(h->copy_out);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

extern "C" int ctd_create(ctd_handle** out, const ctd_config* cfg, const ctd_op* ops, int32_t n_ops,
                          const ctd_bufdesc* bufs, int32_t n_bufs, const void* blob, size_t blob_bytes) {
  ctd_handle* h = nullptr;
  if (!out || !cfg || !ops || !bufs || !blob) return ctd_fail(nullptr, CTD_E_INVALID, "null argument");
  *out = nullptr;
  if (cfg->abi_version != CTD_ABI_VERSION) return ctd_fail(nullptr, CTD_E_INVALID, "ABI version mismatch");
  if (cfg->max_h % 64 || cfg->max_w % 64 || cfg->max_batch < 1) return ctd_fail(nullptr, CTD_E_SHAPE, "bad max shape");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= cfg->device)
    return ctd_fail(nullptr, CTD_E_NO_DEVICE, "no CUDA device %d (this engine has no CPU fallback)", cfg->device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess || prop.major != 9 || prop.minor != 0)
    return ctd_fail(nullptr, CTD_E_NO_DEVICE, "device %d is not sm_90 (compute %d.%d)", cfg->device, prop.major, prop.minor);
  h = new ctd_handle();
  h->cfg = *cfg;
  h->ops.assign(ops, ops + n_ops);
  h->bufs.assign(bufs, bufs + n_bufs);
  {
    // ancestors of the DB tail at buffer granularity (a buffer, once needed, stays needed: several ops may
    // write disjoint channel ranges of it); one backward pass is enough because producers precede consumers
    h->db_ancestor.assign(size_t(n_ops), 0);
    std::vector<char> needed(size_t(n_bufs), 0);
    bool have_db = false;
    for (int i = n_ops - 1; i >= 0; --i) {
      const ctd_op& op = ops[i];
      bool anc = false;
      if (op.kind == CTD_OP_DB_TAIL && !have_db) { anc = true; have_db = true; }
      else if (have_db && op.kind != CTD_OP_DETECT && op.kind != CTD_OP_SEG_TAIL && op.kind != CTD_OP_DB_TAIL) {
        // SPPF_POOL appends its pooled channels to its own source buffer (no dst_buf)
        const int wbuf = op.kind == CTD_OP_SPPF_POOL ? op.src_buf[0] : op.dst_buf;
        anc = wbuf >= 0 && wbuf < n_bufs && needed[wbuf];
      }
      if (!anc) continue;
      h->db_ancestor[size_t(i)] = 1;
      for (int k = 0; k < op.n_src && k < 3; ++k)
        if (op.src_buf[k] >= 0 && op.src_buf[k] < n_bufs) needed[op.src_buf[k]] = 1;
      if (op.residual && op.dst_buf >= 0 && op.dst_buf < n_bufs) needed[op.dst_buf] = 1;
    }
    h->overlap = have_db;
  }
  h->elem = (cfg->precision == CTD_PREC_FP32_SIMT || cfg->precision == CTD_PREC_SPLIT_TC) ? 4 : 2;
  auto bail = [&](int code) { std::string e = h->err; ctd_destroy(h); g_create_error = e; return code; };
  h->detect_prm.assign(size_t(n_ops), {});
  for (int i = 0; i < n_ops; ++i) {
    if (ops[i].kind != CTD_OP_DETECT) continue;
    if (ops[i].p_off < 0 || size_t(ops[i].p_off) + sizeof(h->detect_prm[0]) > blob_bytes) {
      ctd_fail(h, CTD_E_INVALID, "op %d: detect parameters outside the blob", i);
      return bail(CTD_E_INVALID);
    }
    memcpy(h->detect_prm[size_t(i)].data(), static_cast<const char*>(blob) + ops[i].p_off, sizeof(h->detect_prm[0]));
  }
#define CKC(expr)                                                                                        \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) {                                                                             \
      ctd_fail(h, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__);          \
      return bail(CTD_E_CUDA);                                                                           \
    }                                                                                                    \
  } while (0)
  CKC(cudaSetDevice(cfg->device));
  {
    int lo = 0, hi = 0;
    CKC(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    CKC(cudaStreamCreateWithPriority(&h->stream, cudaStreamNonBlocking, lo));
    // side streams get the HIGHER priority: their small blocks slot in whenever a persistent conv CTA retires
    CKC(cudaStreamCreateWithPriority(&h->side, cudaStreamNonBlocking, hi));
    CKC(cudaStreamCreateWithPriority(&h->side2, cudaStreamNonBlocking, hi));
  }
  CKC(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
  CKC(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
  CKC(cudaEventCreateWithFlags(&h->ev_fork2, cudaEventDisableTiming));
  CKC(cudaEventCreateWithFlags(&h->ev_xjoin, cudaEventDisableTiming));
  CKC(cudaEventCreateWithFlags(&h->ev_join2, cudaEventDisableTiming));
  CKC(cudaEventCreateWithFlags(&h->ev_tin, cudaEventDisableTiming));
  CKC(cudaEventCreateWithFlags(&h->ev_tout, cudaEventDisableTiming));
  CKC(cudaEventCreate(&h->ev0));
  CKC(cudaEventCreate(&h->ev1));
  CKC(cudaEventCreate(&h->tev0));
  CKC(cudaEventCreate(&h->tev1));
  {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CKC(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) {
      ctd_fail(h, CTD_E_CUDA, "cuTensorMapEncodeTiled not available from the driver");
      return bail(CTD_E_CUDA);
    }
    h->enc = reinterpret_cast<PFN_encodeTiled>(fn);
  }
  CKC(conv_tc_init());
  CKC(conv_ends_init());
  h->blob_bytes = blob_bytes;
  CKC(cudaMalloc(&h->d_blob, blob_bytes));
  CKC(cudaMemcpy(h->d_blob, blob, blob_bytes, cudaMemcpyHostToDevice));
  const size_t nb = size_t(cfg->max_batch), mh = cfg->max_h, mw = cfg->max_w;
  h->d_buf.assign(n_bufs, nullptr);
  for (int i = 0; i < n_bufs; ++i) {
    const size_t bytes = nb * (mh / bufs[i].down) * (mw / bufs[i].down + 4) * bufs[i].channels * h->elem;
    CKC(cudaMalloc(&h->d_buf[i], bytes));
    CKC(cudaMemset(h->d_buf[i], 0, bytes));
  }
  if (cfg->precision == CTD_PREC_SPLIT_TC) {
    h->d_buf16.assign(n_bufs, nullptr);
    for (int i = 0; i < n_bufs; ++i) {
      const size_t bytes = 2 * nb * (mh / bufs[i].down) * (mw / bufs[i].down + 4) * bufs[i].channels * 2;
      CKC(cudaMalloc(&h->d_buf16[i], bytes));
      CKC(cudaMemset(h->d_buf16[i], 0, bytes));
    }
    // weights: hi rows (the blob's fp16 copy = fp16(w32)) followed by lo rows fp16((w32 - hi) * kSplitLoScale),
    // per GEMM op
    h->wsplit_off.assign(size_t(n_ops), 0);
    std::vector<__half> ws;
    const char* hb = static_cast<const char*>(blob);
    for (int i = 0; i < n_ops; ++i) {
      const ctd_op& op = ops[i];
      if (!is_gemm(op.kind)) continue;
      int cin = 0;
      for (int k = 0; k < op.n_src; ++k) cin += op.src_c[k];
      const int taps = op.kind == CTD_OP_DECONV4 ? 4 : op.ksize * op.ksize;
      const int nph = op.kind == CTD_OP_DECONV4 ? 4 : 1;
      const size_t cnt = size_t(nph) * op.cout_pad * taps * cin;
      if (size_t(op.w32_off) + cnt * 4 > blob_bytes || size_t(op.w16_off) + cnt * 2 > blob_bytes) {
        ctd_fail(h, CTD_E_INVALID, "op %d: weights outside the blob", i);
        return bail(CTD_E_INVALID);
      }
      while (ws.size() % 128) ws.push_back(__float2half(0.f));   // 256-byte aligned rows for the tensor map
      h->wsplit_off[size_t(i)] = ws.size() * 2;
      const float* w32 = reinterpret_cast<const float*>(hb + op.w32_off);
      const size_t base = ws.size();
      ws.resize(base + 2 * cnt);
      for (size_t k = 0; k < cnt; ++k) {
        const __half hi = __float2half_rn(w32[k]);
        ws[base + k] = hi;
        ws[base + cnt + k] = __float2half_rn((w32[k] - __half2float(hi)) * kSplitLoScale);
      }
    }
    CKC(cudaMalloc(&h->d_wsplit, ws.size() * 2 + 256));
    CKC(cudaMemcpy(h->d_wsplit, ws.data(), ws.size() * 2, cudaMemcpyHostToDevice));
  }
  const size_t px = nb * mh * mw;
  const int no = 5 + cfg->nc;
  CKC(cudaMalloc(&h->d_pages, px * 3));
  CKC(cudaMalloc(&h->d_blks, nb * rows_per_image(mh, mw) * no * sizeof(float)));
  CKC(cudaMalloc(&h->d_mask, px * 4));
  CKC(cudaMalloc(&h->d_lines, px * 2 * 4));
  CKC(cudaMalloc(&h->d_bitmap, px));
  CKC(cudaMalloc(&h->d_labels, px * 4));
  {
    auto al = [](size_t v) { return (v + 255) / 256 * 256; };
    ArenaLayout& L = h->layout;
    L.det = al(px); L.cnt = L.det + al(nb * 300 * 6 * 4); L.nl = L.cnt + al(nb * 4);
    L.lb = L.nl + al(nb * 4); L.ls = L.lb + al(nb * 1000 * 8 * 2); L.lc = L.ls + al(nb * 1000 * 4);
    L.a_bytes = L.lc + al(nb * 4);
    L.refined = L.a_bytes;
    L.blocks = L.refined + al(px);
    const BlockSection bs = block_section_layout();
    L.rec_off = bs.rec_off; L.lines_off = bs.lines_off; L.dist_off = bs.dist_off; L.blocks_stride = bs.stride;
    L.total = L.blocks + nb * L.blocks_stride;
    CKC(cudaMalloc(&h->d_mask_u8, L.total));
    CKC(cudaMemset(h->d_mask_u8, 0, L.total));
    h->d_det = reinterpret_cast<float*>(h->d_mask_u8 + L.det);
    h->d_det_count = reinterpret_cast<int*>(h->d_mask_u8 + L.cnt);
    h->d_nlabels = reinterpret_cast<int32_t*>(h->d_mask_u8 + L.nl);
    h->d_line_boxes = reinterpret_cast<int16_t*>(h->d_mask_u8 + L.lb);
    h->d_line_scores = reinterpret_cast<float*>(h->d_mask_u8 + L.ls);
    h->d_line_count = reinterpret_cast<int32_t*>(h->d_mask_u8 + L.lc);
  }
  CKC(cudaMalloc(&h->d_ccl_scratch, px * 4 * 3));
  CKC(cudaMalloc(&h->d_segrep_scratch, segrep_scratch_bytes(int(nb), int(mh), int(mw), 1000)));
  {
    // n x h of the largest launch: a batch, or one ctd_seg_represent map of up to 2048 rows
    const size_t rows_bytes = std::max(nb * mh, size_t(2048)) * 1000 * sizeof(int2);
    CKC(cudaMalloc(&h->d_segrep_rows, rows_bytes));
    CKC(cudaMemset(h->d_segrep_rows, 0xff, rows_bytes));
  }
  const int cap = 4096;
  CKC(cudaMalloc(&h->d_nms_ws, nms_workspace_bytes(int(nb), cap)));
  nms_workspace_bind(h->nms, h->d_nms_ws, int(nb), cap);
  CKC(cudaDeviceSynchronize());
#undef CKC
  *out = h;
  return CTD_OK;
}

// -----------------------------------------------------------------------------------------
static int op_geom(ctd_handle* h, const ctd_op& op, int n, int ph, int pw, ConvGeom& g) {
  memset(&g, 0, sizeof(g));
  fill_conv_geom_taps(g, op.kind == CTD_OP_DETECT ? CTD_OP_CONV : op.kind, op.ksize, op.stride);
  g.n_img = n;
  g.n_src = op.n_src;
  const ctd_bufdesc& sb = h->bufs[op.src_buf[0]];
  g.src_h = ph / sb.down;
  g.src_w = pw / sb.down;
  g.cin_total = 0;
  for (int s = 0; s < op.n_src; ++s) {
    const ctd_bufdesc& b = h->bufs[op.src_buf[s]];
    if (b.down != sb.down) return ctd_fail(h, CTD_E_INVALID, "op sources differ in resolution");
    g.src_c[s] = op.src_c[s];
    g.src_cstride[s] = b.channels;
    g.cin_total += op.src_c[s];
  }
  g.k_total = g.taps * g.cin_total;
  g.gh = op.kind == CTD_OP_DECONV4 ? g.src_h : g.src_h / op.stride;
  g.gw = op.kind == CTD_OP_DECONV4 ? g.src_w : g.src_w / op.stride;
  g.dst_h = g.gh * g.out_mul;
  g.dst_w = g.gw * g.out_mul;
  g.cout = op.cout;
  g.cout_pad = op.cout_pad;
  if (op.dst_buf >= 0) {
    g.dst_cstride = h->bufs[op.dst_buf].channels;
    g.dst_coff = op.dst_coff;
  }
  g.act = op.act;
  g.residual = op.residual;
  return CTD_OK;
}

// DETECT epilogue: the decoded rows of pyramid level op.aux go to d_blks (ConvTcParams and ConvSimtParams)
template <typename P>
static void set_detect(const ctd_handle* h, size_t i, int ph, int pw, P& p) {
  p.blks = h->d_blks;
  p.blks_rows_per_img = rows_per_image(ph, pw);
  int row0 = 0;
  for (int l = 0; l < h->ops[i].aux; ++l) row0 += 3 * (ph / (8 << l)) * (pw / (8 << l));
  p.level_row0 = row0;
  p.nc = h->cfg.nc;
  p.det_stride = h->detect_prm[i][0];
  for (int k = 0; k < 6; ++k) p.anchor_wh[k] = h->detect_prm[i][1 + k];
}

// Ops that run on the tensor cores (conv_tc_kernel, or the stem / seg-tail kernels); every other op runs on the CUDA
// cores.
static bool runs_on_tensor_cores(int precision, int kind) {
  switch (precision) {
    case CTD_PREC_SPLIT_TC: return is_gemm(kind);
    case CTD_PREC_FP16_TC: return is_gemm(kind) || kind == CTD_OP_STEM || kind == CTD_OP_SEG_TAIL;
    default: return false;
  }
}

// tensor-core launch plans of one shape: the only place that picks an op's kernel by precision
static int build_plans(ctd_handle* h, int n, int ph, int pw, ShapePlan& sp) {
  sp.tc.resize(h->ops.size());
  sp.ends.resize(h->ops.size());
  const bool split = h->cfg.precision == CTD_PREC_SPLIT_TC;
  for (size_t i = 0; i < h->ops.size(); ++i) {
    const ctd_op& op = h->ops[i];
    if (!runs_on_tensor_cores(h->cfg.precision, op.kind)) continue;
    const float* bias = reinterpret_cast<const float*>(h->d_blob + op.b_off);
    const char* e = nullptr;
    if (op.kind == CTD_OP_STEM) {
      // reads the u8 pages (or the fp16 staging page of a float input) itself: the space-to-depth form is built per
      // tile in shared memory
      const bool f16 = sp.input == INPUT_F32;
      e = conv_ends_plan_stem(sp.ends[i], h->enc, f16 ? static_cast<const void*>(h->in_stage.p) : h->d_pages, f16, n,
                              ph, pw, h->d_blob + op.w16_off, bias, static_cast<__half*>(h->d_buf[op.dst_buf]),
                              h->bufs[op.dst_buf].channels, op.dst_coff, op.cout, op.act);
    } else if (op.kind == CTD_OP_SEG_TAIL) {
      // the final ConvT 4x4 s2 (C -> 1) as a 3x3 convolution whose 4 output channels are the sub-pixel phases, with
      // the sigmoid / u8-mask epilogue
      if (op.cout_pad != 16) return ctd_fail(h, CTD_E_INVALID, "op %zu: seg tail needs cout_pad 16", i);
      const ctd_bufdesc& sb = h->bufs[op.src_buf[0]];
      e = conv_ends_plan_seg(sp.ends[i], h->enc, static_cast<const __half*>(h->d_buf[op.src_buf[0]]), sb.channels,
                             op.src_coff[0], op.src_c[0], n, ph / sb.down, pw / sb.down, h->d_blob + op.w16_off,
                             h->d_mask, h->d_mask_u8);
    } else {
      ConvGeom g;
      if (int rc = op_geom(h, op, n, ph, pw, g)) return rc;
      const void* src[CTD_MAX_SRC];
      int coff[CTD_MAX_SRC];
      for (int s = 0; s < op.n_src; ++s) {
        src[s] = (split ? h->d_buf16 : h->d_buf)[op.src_buf[s]];
        coff[s] = op.src_coff[s];
      }
      const void* w = split ? h->d_wsplit + h->wsplit_off[i] : h->d_blob + op.w16_off;
      __half* dst = op.kind == CTD_OP_DETECT ? nullptr : static_cast<__half*>(h->d_buf[op.dst_buf]);
      e = conv_tc_plan(sp.tc[i], h->enc, g, src, coff, w, bias, dst, split);
      if (op.kind == CTD_OP_DETECT) set_detect(h, i, ph, pw, sp.tc[i].p);
    }
    if (e) return ctd_fail(h, CTD_E_INVALID, "op %zu: %s", i, e);
  }
  return CTD_OK;
}

template <typename T>
static int run_op_simt(ctd_handle* h, size_t i, int n, int ph, int pw) {
  const ctd_op& op = h->ops[i];
  ConvSimtParams p;
  memset(&p, 0, sizeof(p));
  if (int rc = op_geom(h, op, n, ph, pw, p.g)) return rc;
  for (int k = 0; k < op.n_src; ++k)
    p.src[k] = static_cast<char*>(h->d_buf[op.src_buf[k]]) + size_t(op.src_coff[k]) * sizeof(T);
  p.w = h->d_blob + (sizeof(T) == 4 ? op.w32_off : op.w16_off);
  p.bias = reinterpret_cast<const float*>(h->d_blob + op.b_off);
  if (op.kind == CTD_OP_DETECT) set_detect(h, i, ph, pw, p);
  else p.dst = h->d_buf[op.dst_buf];
  CK(conv_simt_launch<T>(p, h->stream));
  return CTD_OK;
}

template <typename T>
static int run_op_thin(ctd_handle* h, const ctd_op& op, int n, int ph, int pw, int input) {
  cudaStream_t s = h->stream;
  const ctd_bufdesc* sb = op.kind == CTD_OP_STEM ? nullptr : &h->bufs[op.src_buf[0]];
  const int sh = sb ? ph / sb->down : ph, sw = sb ? pw / sb->down : pw;
  const T* src = sb ? static_cast<const T*>(h->d_buf[op.src_buf[0]]) + op.src_coff[0] : nullptr;
  switch (op.kind) {
    case CTD_OP_STEM: {
      const float* w = reinterpret_cast<const float*>(h->d_blob + op.w32_off);
      const float* b = reinterpret_cast<const float*>(h->d_blob + op.b_off);
      T* dst = static_cast<T*>(h->d_buf[op.dst_buf]);
      const int dc = h->bufs[op.dst_buf].channels;
      if (input == INPUT_U8) {
        CK(stem_launch<T>(h->d_pages, n, ph, pw, w, b, dst, dc, op.dst_coff, op.cout, op.act, s));
      } else {   // the f32 staging page: the fp16 tensor-core engine runs its stem in stem_tc_kernel
        CK(stem_launch<T>(reinterpret_cast<const float*>(h->in_stage.p), n, ph, pw, w, b, dst, dc, op.dst_coff,
                          op.cout, op.act, s));
      }
      return CTD_OK;
    }
    case CTD_OP_AVGPOOL2:
      CK(avgpool2_launch<T>(src, n, sh, sw, op.src_c[0], sb->channels,
                            static_cast<T*>(h->d_buf[op.dst_buf]) + op.dst_coff, h->bufs[op.dst_buf].channels, s));
      return CTD_OK;
    case CTD_OP_SPPF_POOL:
      CK(sppf_pool_launch<T>(static_cast<T*>(h->d_buf[op.src_buf[0]]) + op.src_coff[0], n, sh, sw, op.src_c[0],
                             sb->channels, s));
      return CTD_OK;
    case CTD_OP_UPSAMPLE2:
      CK(upsample2_launch<T>(src, n, sh, sw, op.src_c[0], sb->channels,
                             static_cast<T*>(h->d_buf[op.dst_buf]) + op.dst_coff, h->bufs[op.dst_buf].channels, s));
      return CTD_OK;
    case CTD_OP_SEG_TAIL:
      CK(seg_tail_launch<T>(src, n, sh, sw, op.src_c[0], sb->channels,
                            reinterpret_cast<const float*>(h->d_blob + op.p_off), h->d_mask, h->d_mask_u8, s));
      return CTD_OK;
    case CTD_OP_DB_TAIL:
      CK(db_tail_launch<T>(src, n, sh, sw, sb->channels, reinterpret_cast<const float*>(h->d_blob + op.p_off),
                           h->d_lines, h->d_bitmap, h->cfg.db_thresh, s));
      return CTD_OK;
    default: return ctd_fail(h, CTD_E_INVALID, "run_op_thin: bad kind %d", op.kind);
  }
}

// split-fp16 mode: refresh the fp16 hi | lo planes of the channel slice op `i` has just written
static int split_written_slice(ctd_handle* h, const ctd_op& op, int n, int ph, int pw, int* cnt) {
  int buf = op.dst_buf, coff = op.dst_coff, c = op.cout;
  if (op.kind == CTD_OP_SPPF_POOL) { buf = op.src_buf[0]; coff = op.src_coff[0] + op.src_c[0]; c = 3 * op.src_c[0]; }
  else if (op.kind == CTD_OP_AVGPOOL2 || op.kind == CTD_OP_UPSAMPLE2) c = op.src_c[0];
  if (buf < 0 || c <= 0) return CTD_OK;
  const ctd_bufdesc& b = h->bufs[buf];
  const size_t npix = size_t(n) * (ph / b.down) * (pw / b.down);
  __half* hi = static_cast<__half*>(h->d_buf16[buf]) + coff;
  CK(split_planes_launch(static_cast<const float*>(h->d_buf[buf]) + coff, hi, hi + npix * b.channels, npix, c, b.channels,
                         h->stream));
  ++*cnt;
  return CTD_OK;
}

static int run_one_op(ctd_handle* h, size_t i, int n, int ph, int pw, const ShapePlan& sp, int* cnt) {
  const ctd_op& op = h->ops[i];
  const ConvTcPlan& tc = sp.tc[i];
  int rc = CTD_OK;
  if (tc.block_n || sp.ends[i].kind != ctd::CTD_END_NONE) {
    const cudaError_t e = tc.block_n ? conv_tc_launch(tc, h->stream) : conv_ends_launch(sp.ends[i], h->stream);
    if (e != cudaSuccess) rc = ctd_fail(h, CTD_E_CUDA, "tensor-core op %zu: %s", i, cudaGetErrorString(e));
  } else if (is_gemm(op.kind)) {
    rc = h->elem == 4 ? run_op_simt<float>(h, i, n, ph, pw) : run_op_simt<__half>(h, i, n, ph, pw);
  } else {
    rc = h->elem == 4 ? run_op_thin<float>(h, op, n, ph, pw, sp.input) : run_op_thin<__half>(h, op, n, ph, pw, sp.input);
  }
  ++*cnt;
  if (rc || h->d_buf16.empty()) return rc;
  return split_written_slice(h, op, n, ph, pw, cnt);   // split-fp16 mode: refresh the planes of what the op wrote
}

// NMS of the Detect rows
int launch_nms(ctd_handle* h, int n, int ph, int pw, cudaStream_t s, int* cnt, const int32_t* half) {
  CK(nms_launch(h->d_blks, n, rows_per_image(ph, pw), h->cfg.nc, h->cfg.conf_thresh, h->cfg.nms_thresh, h->nms, h->d_det,
                h->d_det_count, s, half));
  *cnt += kNmsLaunches;
  return CTD_OK;
}

// DB post-processing: connected components of the bitmap, then the text-line boxes.  The label plane numbered like
// OpenCV is built only when ctd_get_db_components asks for it.
int launch_db_post(ctd_handle* h, int n, int ph, int pw, cudaStream_t s, int* cnt) {
  CK(ccl_launch(h->d_bitmap, n, ph, pw, h->d_ccl_scratch, h->d_nlabels, s));
  CK(segrep_launch(h->d_bitmap, h->d_lines, size_t(2) * ph * pw, h->d_ccl_scratch, n, ph, pw, 1000, 1.5f,
                   h->d_segrep_scratch, h->d_segrep_rows, h->d_line_boxes, h->d_line_scores, h->d_line_count, s));
  *cnt += kCclLaunches + kSegrepLaunches;
  return CTD_OK;
}

static int run_ops(ctd_handle* h, int n, int ph, int pw, const ShapePlan& sp, int* launches, bool record = false) {
  int cnt = 0;
  size_t evi = 0;
  if (h->overlap && !record && !h->cfg.debug_skip_postproc) {
    // Two-phase order.  Phase 1: every op the DB maps depend on (program order).  Then the DB post-processing
    // (CCL + contour boxes: latency-bound kernels that leave most SMs idle) forks to a side stream and runs
    // UNDER phase 2 = the rest of the network (PAN, Detect heads, the seg-head tail); NMS forks the same way once
    // the Detect rows exist.  No buffer is shared between the branches (the compiler never reuses buffers).
    for (size_t i = 0; i < h->ops.size(); ++i)
      if (h->db_ancestor[i])
        if (int rc = run_one_op(h, i, n, ph, pw, sp, &cnt)) return rc;
    CK(cudaEventRecord(h->ev_fork, h->stream));
    CK(cudaStreamWaitEvent(h->side, h->ev_fork, 0));
    if (int rc = launch_db_post(h, n, ph, pw, h->side, &cnt)) return rc;
    CK(cudaEventRecord(h->ev_join, h->side));
    size_t last_detect = h->ops.size();
    for (size_t i = 0; i < h->ops.size(); ++i)
      if (!h->db_ancestor[i] && h->ops[i].kind == CTD_OP_DETECT) last_detect = i;
    bool nms_forked = false;
    for (size_t i = 0; i < h->ops.size(); ++i) {   // program order: PAN -> Detect heads -> seg-head tail
      if (h->db_ancestor[i]) continue;
      if (int rc = run_one_op(h, i, n, ph, pw, sp, &cnt)) return rc;
      if (i == last_detect) {
        CK(cudaEventRecord(h->ev_fork2, h->stream));
        CK(cudaStreamWaitEvent(h->side2, h->ev_fork2, 0));
        if (int rc = launch_nms(h, n, ph, pw, h->side2, &cnt)) return rc;
        CK(cudaEventRecord(h->ev_join2, h->side2));
        nms_forked = true;
      }
    }
    if (!nms_forked) {
      if (int rc = launch_nms(h, n, ph, pw, h->stream, &cnt)) return rc;
    } else {
      CK(cudaStreamWaitEvent(h->stream, h->ev_join2, 0));
    }
    CK(cudaStreamWaitEvent(h->stream, h->ev_join, 0));
    *launches = cnt;
    return CTD_OK;
  }
  if (record) CK(cudaEventRecord(h->op_events[evi++], h->stream));
  for (size_t i = 0; i < h->ops.size(); ++i) {
    if (int rc = run_one_op(h, i, n, ph, pw, sp, &cnt)) return rc;
    if (record) CK(cudaEventRecord(h->op_events[evi++], h->stream));
  }
  *launches = cnt;
  if (h->cfg.debug_skip_postproc) return CTD_OK;
  // post-processing on the same stream
  if (int rc = launch_nms(h, n, ph, pw, h->stream, &cnt)) return rc;
  if (record) CK(cudaEventRecord(h->op_events[evi++], h->stream));
  if (int rc = launch_db_post(h, n, ph, pw, h->stream, &cnt)) return rc;
  if (record) CK(cudaEventRecord(h->op_events[evi++], h->stream));
  *launches = cnt;
  return CTD_OK;
}

// bytes per element of ctd_forward_tensor's staging page: fp16 for the fp16 tensor-core stem, f32 for the CUDA-core stem
static size_t stage_elem(const ctd_handle* h) { return h->cfg.precision == CTD_PREC_FP16_TC ? 2 : 4; }

// shape checks + the launch plans of (n, ph, pw, input), built on first use
static int find_plan(ctd_handle* h, int32_t n, int32_t ph, int32_t pw, ShapePlan** out, int input = INPUT_U8) {
  if (n < 1 || n > h->cfg.max_batch) return ctd_fail(h, CTD_E_CAPACITY, "batch %d exceeds max_batch %d", n, h->cfg.max_batch);
  if (ph % 64 || pw % 64 || ph > h->cfg.max_h || pw > h->cfg.max_w || ph < 64 || pw < 64)
    return ctd_fail(h, CTD_E_SHAPE, "page %dx%d must be a multiple of 64 and <= %dx%d", ph, pw, h->cfg.max_h, h->cfg.max_w);
  CK(cudaSetDevice(h->cfg.device));
  auto key = std::make_tuple(int(n), int(ph), int(pw), input);
  auto it = h->plans.find(key);
  if (it == h->plans.end()) {
    ShapePlan sp;
    sp.input = input;
    if (input == INPUT_F32) {
      // the whole workspace at once: the page never moves, so every plan's tensor map and captured graph stays valid
      const size_t bytes = size_t(h->cfg.max_batch) * h->cfg.max_h * h->cfg.max_w * 3 * stage_elem(h);
      if (int rc = h->in_stage.grow(h, bytes, std::nullopt, size_t(1) << 40)) return rc;
    }
    if (int rc = build_plans(h, n, ph, pw, sp)) return rc;
    it = h->plans.emplace(key, std::move(sp)).first;
  }
  *out = &it->second;
  return CTD_OK;
}

// plan lookup + (first time, use_graph) graph capture; the forward itself is enqueue_forward()
int prepare_forward(ctd_handle* h, int32_t n, int32_t ph, int32_t pw, ShapePlan** out, int input) {
  ShapePlan* sp = nullptr;
  if (int rc = find_plan(h, n, ph, pw, &sp, input)) return rc;
  if (h->cfg.use_graph && !sp->graph) {
    cudaGraph_t graph;
    CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    int rc = run_ops(h, n, ph, pw, *sp, &sp->launches);
    cudaError_t e = cudaStreamEndCapture(h->stream, &graph);
    if (rc) return rc;
    CK(e);
    CK(cudaGraphInstantiate(&sp->graph, graph, 0));
    cudaGraphDestroy(graph);
  }
  *out = sp;
  return CTD_OK;
}

int enqueue_forward(ctd_handle* h, int32_t n, int32_t ph, int32_t pw, ShapePlan& sp) {
  if (sp.graph) {
    CK(cudaGraphLaunch(sp.graph, h->stream));
  } else {
    if (int rc = run_ops(h, n, ph, pw, sp, &sp.launches)) return rc;
  }
  CK(cudaEventRecord(h->ev1, h->stream));
  h->last_launches = sp.launches;
  h->n = n; h->ph = ph; h->pw = pw;
  h->have_forward = true;
  return CTD_OK;
}

extern "C" int ctd_forward(ctd_handle* h, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw,
                           int32_t pages_on_device) {
  if (!h || !pages) return CTD_E_INVALID;
  ShapePlan* sp = nullptr;
  if (int rc = prepare_forward(h, n, ph, pw, &sp)) return rc;
  const size_t bytes = size_t(n) * ph * pw * 3;
  CK(cudaEventRecord(h->ev0, h->stream));
  CK(cudaMemcpyAsync(h->d_pages, pages, bytes, pages_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                     h->stream));
  return enqueue_forward(h, n, ph, pw, *sp);
}

// float32 -> T, round to nearest even for __half
template <typename T>
__global__ void from_f32_kernel(const float* src, T* dst, size_t n) {
  size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x;
  if (i < n) dst[i] = T(src[i]);
}

// a workspace output of the forward into the caller's tensor: a copy (X = float), or rounded to nearest even (__half)
template <typename X>
static int copy_output(ctd_handle* h, X* dst, const float* src, size_t elems) {
  if constexpr (sizeof(X) == 4) {
    CK(cudaMemcpyAsync(dst, src, elems * 4, cudaMemcpyDeviceToDevice, h->stream));
  } else {
    from_f32_kernel<__half><<<unsigned((elems + 255) / 256), 256, 0, h->stream>>>(src, dst, elems);
    CK(cudaGetLastError());
  }
  return CTD_OK;
}

// ctd_forward_tensor (X = float) and ctd_forward_tensor_f16 (X = __half): the input pre-pass from an X tensor, the
// forward, and the outputs as X
template <typename X>
static int forward_tensor(ctd_handle* h, const X* x, int32_t n, int32_t ph, int32_t pw, void* stream, X* blks, X* mask,
                          X* lines) {
  if (!h || !x) return CTD_E_INVALID;
  if (reinterpret_cast<uintptr_t>(x) % 16) return ctd_fail(h, CTD_E_INVALID, "x must be 16-byte aligned");
  ShapePlan* sp = nullptr;
  if (int rc = prepare_forward(h, n, ph, pw, &sp, INPUT_F32)) return rc;
  cudaStream_t cs = static_cast<cudaStream_t>(stream);
  CK(cudaEventRecord(h->ev_tin, cs));   // x and the outputs are ready for the engine once the caller's work so far ran
  CK(cudaStreamWaitEvent(h->stream, h->ev_tin, 0));
  CK(cudaEventRecord(h->ev0, h->stream));
  if (stage_elem(h) == 2)
    CK(nchw_to_hwc_launch(x, n, ph, pw, reinterpret_cast<__half*>(h->in_stage.p), h->stream));
  else
    CK(nchw_to_hwc_launch(x, n, ph, pw, reinterpret_cast<float*>(h->in_stage.p), h->stream));
  if (int rc = enqueue_forward(h, n, ph, pw, *sp)) return rc;
  const size_t px = size_t(n) * ph * pw;
  if (blks)
    if (int rc = copy_output(h, blks, h->d_blks, size_t(n) * rows_per_image(ph, pw) * (5 + h->cfg.nc))) return rc;
  if (mask)
    if (int rc = copy_output(h, mask, h->d_mask, px)) return rc;
  if (lines)
    if (int rc = copy_output(h, lines, h->d_lines, px * 2)) return rc;
  CK(cudaEventRecord(h->ev_tout, h->stream));
  CK(cudaStreamWaitEvent(cs, h->ev_tout, 0));
  return CTD_OK;
}

extern "C" int ctd_forward_tensor(ctd_handle* h, const float* x, int32_t n, int32_t ph, int32_t pw, void* stream,
                                  float* blks, float* mask, float* lines) {
  return forward_tensor(h, x, n, ph, pw, stream, blks, mask, lines);
}

extern "C" int ctd_forward_tensor_f16(ctd_handle* h, const void* x, int32_t n, int32_t ph, int32_t pw, void* stream,
                                      void* blks, void* mask, void* lines) {
  return forward_tensor(h, static_cast<const __half*>(x), n, ph, pw, stream, static_cast<__half*>(blks),
                        static_cast<__half*>(mask), static_cast<__half*>(lines));
}

template <bool kPinned>
int GrowBuf<kPinned>::grow(ctd_handle* h, size_t bytes, std::optional<cudaStream_t> sync, size_t headroom) {
  if (bytes <= cap) return CTD_OK;
  if (sync) CK(cudaStreamSynchronize(*sync));
  release();
  const size_t alloc = bytes + bytes / headroom;
  if (kPinned) CK(cudaHostAlloc(reinterpret_cast<void**>(&p), alloc, cudaHostAllocDefault));
  else CK(cudaMalloc(reinterpret_cast<void**>(&p), alloc));
  cap = alloc;
  return CTD_OK;
}
template <bool kPinned>
void GrowBuf<kPinned>::release() {
  if (kPinned && p) cudaFreeHost(p);
  if (!kPinned) cudaFree(p);
  p = nullptr;
  cap = 0;
}
template struct GrowBuf<false>;
template struct GrowBuf<true>;

void Slot::release() {
  cudaFree(d_stage_in);
  cudaFree(d_stage_out);
  for (cudaEvent_t e : {ev_in_done, ev_in_free, ev_out_ready, ev_out_done, ev_post_done})
    if (e) cudaEventDestroy(e);
  if (pinned) cudaFreeHost(pinned);
  pg_in.release(); pg_res.release(); pg_aux.release(); out_in.release(); d_crop.release(); h_crop.release();
  cudaFree(d_pg_tab);
  if (h_pg_tab) cudaFreeHost(h_pg_tab);
  *this = Slot();
}

extern "C" int ctd_resize_linear_u8(ctd_handle* h, const uint8_t* src, int32_t sh, int32_t sw, int32_t channels, uint8_t* dst,
                                    int32_t dh, int32_t dw) {
  if (!h || !src || !dst) return CTD_E_INVALID;
  if ((channels != 1 && channels != 3) || sh < 1 || sw < 1 || dh < 1 || dw < 1) return ctd_fail(h, CTD_E_SHAPE, "bad resize shape");
  CK(cudaSetDevice(h->cfg.device));
  const size_t sb = size_t(sh) * sw * channels, db = size_t(dh) * dw * channels;
  const size_t so = (sb + 255) / 256 * 256;
  if (int rc = h->io_scratch.grow(h, so + db, h->stream)) return rc;
  CK(cudaMemcpyAsync(h->io_scratch.p, src, sb, cudaMemcpyHostToDevice, h->stream));
  CK(resize_linear_u8_launch(h->io_scratch.p, sh, sw, size_t(sw) * channels, channels, h->io_scratch.p + so, dh, dw, dh, dw, h->stream));
  CK(cudaMemcpyAsync(dst, h->io_scratch.p + so, db, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_join(ctd_handle* h, ctd_handle* other) {
  if (!h || !other) return CTD_E_INVALID;
  if (h == other) return CTD_OK;
  if (h->cfg.device != other->cfg.device) return ctd_fail(h, CTD_E_INVALID, "ctd_join: handles live on different devices");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventRecord(other->ev_xjoin, other->stream));
  CK(cudaStreamWaitEvent(h->stream, other->ev_xjoin, 0));
  return CTD_OK;
}

#define NEED_FWD()                                                                     \
  if (!h) return CTD_E_INVALID;                                                        \
  if (!h->have_forward) return ctd_fail(h, CTD_E_INVALID, "no forward pass has been run"); \
  CK(cudaSetDevice(h->cfg.device));

extern "C" int ctd_get_net_outputs(ctd_handle* h, float* blks, float* mask, float* lines) {
  NEED_FWD();
  const size_t px = size_t(h->n) * h->ph * h->pw;
  if (blks)
    CK(cudaMemcpyAsync(blks, h->d_blks, size_t(h->n) * rows_per_image(h->ph, h->pw) * (5 + h->cfg.nc) * 4,
                       cudaMemcpyDeviceToHost, h->stream));
  if (mask) CK(cudaMemcpyAsync(mask, h->d_mask, px * 4, cudaMemcpyDeviceToHost, h->stream));
  if (lines) CK(cudaMemcpyAsync(lines, h->d_lines, px * 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_get_mask_u8(ctd_handle* h, uint8_t* mask_u8) {
  NEED_FWD();
  if (!mask_u8) return CTD_E_INVALID;
  CK(cudaMemcpyAsync(mask_u8, h->d_mask_u8, size_t(h->n) * h->ph * h->pw, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_get_detections(ctd_handle* h, float* det, int32_t* det_count) {
  NEED_FWD();
  if (!det || !det_count) return CTD_E_INVALID;
  CK(cudaMemcpyAsync(det, h->d_det, size_t(h->n) * 300 * 6 * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(det_count, h->d_det_count, size_t(h->n) * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_get_nms_status(ctd_handle* h, int32_t* cand_total, int32_t* cap) {
  if (!h) return CTD_E_INVALID;
  CK(cudaSetDevice(h->cfg.device));
  if (cap) *cap = h->nms.cap;
  if (cand_total) {
    const int n = h->have_forward ? h->n : 1;
    CK(cudaMemcpyAsync(cand_total, h->nms.cand_total, size_t(n) * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return CTD_OK;
}

extern "C" int ctd_get_db_components(ctd_handle* h, uint8_t* bitmap, int32_t* labels, int32_t* n_labels) {
  NEED_FWD();
  const size_t px = size_t(h->n) * h->ph * h->pw;
  if (bitmap) CK(cudaMemcpyAsync(bitmap, h->d_bitmap, px, cudaMemcpyDeviceToHost, h->stream));
  if (labels) {
    CK(ccl_number_launch(h->n, h->ph, h->pw, h->d_ccl_scratch, h->d_labels, h->stream));
    CK(cudaMemcpyAsync(labels, h->d_labels, px * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  if (n_labels) CK(cudaMemcpyAsync(n_labels, h->d_nlabels, size_t(h->n) * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_get_text_lines(ctd_handle* h, int16_t* boxes, float* scores, int32_t* counts) {
  NEED_FWD();
  if (!boxes || !scores || !counts) return CTD_E_INVALID;
  CK(cudaMemcpyAsync(boxes, h->d_line_boxes, size_t(h->n) * 1000 * 8 * 2, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(scores, h->d_line_scores, size_t(h->n) * 1000 * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(counts, h->d_line_count, size_t(h->n) * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_seg_represent(ctd_handle* h, const float* pred, int32_t ih, int32_t iw, float thresh, int16_t* boxes,
                                 float* scores, int32_t* count) {
  if (!h || !pred || !boxes || !scores || !count) return CTD_E_INVALID;
  if (ih < 1 || iw < 1 || size_t(ih) * iw > size_t(h->cfg.max_h) * h->cfg.max_w || ih > 2048 || iw > 2048)
    return ctd_fail(h, CTD_E_CAPACITY, "map larger than the workspace");
  CK(cudaSetDevice(h->cfg.device));
  const size_t px = size_t(ih) * iw;
  CK(cudaMemcpyAsync(h->d_lines, pred, px * 4, cudaMemcpyHostToDevice, h->stream));
  CK(binarize_launch(h->d_lines, px, thresh, h->d_bitmap, h->stream));
  CK(ccl_launch(h->d_bitmap, 1, ih, iw, h->d_ccl_scratch, h->d_nlabels, h->stream));
  CK(segrep_launch(h->d_bitmap, h->d_lines, px, h->d_ccl_scratch, 1, ih, iw, 1000, 1.5f, h->d_segrep_scratch,
                   h->d_segrep_rows, h->d_line_boxes, h->d_line_scores, h->d_line_count, h->stream));
  CK(cudaMemcpyAsync(boxes, h->d_line_boxes, 1000 * 8 * 2, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(scores, h->d_line_scores, 1000 * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(count, h->d_line_count, 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->have_forward = false;
  return CTD_OK;
}

extern "C" int ctd_last_forward_ms(ctd_handle* h, float* ms) {
  NEED_FWD();
  if (!ms) return CTD_E_INVALID;
  CK(cudaEventSynchronize(h->ev1));
  CK(cudaEventElapsedTime(ms, h->ev0, h->ev1));
  return CTD_OK;
}

extern "C" int ctd_last_launch_count(ctd_handle* h, int32_t* launches) {
  NEED_FWD();
  if (!launches) return CTD_E_INVALID;
  *launches = h->last_launches;
  return CTD_OK;
}

extern "C" int ctd_timer_start(ctd_handle* h) {
  if (!h) return CTD_E_INVALID;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventRecord(h->tev0, h->stream));
  return CTD_OK;
}
extern "C" int ctd_timer_stop(ctd_handle* h, float* ms) {
  if (!h || !ms) return CTD_E_INVALID;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventRecord(h->tev1, h->stream));
  CK(cudaEventSynchronize(h->tev1));
  CK(cudaEventElapsedTime(ms, h->tev0, h->tev1));
  return CTD_OK;
}

extern "C" int ctd_profile_forward(ctd_handle* h, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw,
                                   int32_t pages_on_device, float* op_ms, int32_t cap) {
  if (!h || !pages || !op_ms) return CTD_E_INVALID;
  const int need = int(h->ops.size()) + 2;
  if (cap < need) return ctd_fail(h, CTD_E_INVALID, "op_ms needs %d entries", need);
  ShapePlan* sp = nullptr;
  if (int rc = find_plan(h, n, ph, pw, &sp)) return rc;
  while (int(h->op_events.size()) < need + 1) {
    cudaEvent_t e;
    CK(cudaEventCreate(&e));
    h->op_events.push_back(e);
  }
  CK(cudaMemcpyAsync(h->d_pages, pages, size_t(n) * ph * pw * 3,
                     pages_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
  int launches = 0;
  if (int rc = run_ops(h, n, ph, pw, *sp, &launches, true)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  const int nev = h->cfg.debug_skip_postproc ? int(h->ops.size()) : need;
  for (int i = 0; i < need; ++i) op_ms[i] = 0.f;
  for (int i = 0; i < nev; ++i) CK(cudaEventElapsedTime(&op_ms[i], h->op_events[i], h->op_events[i + 1]));
  h->n = n; h->ph = ph; h->pw = pw;
  h->have_forward = true;
  h->last_launches = launches;
  return CTD_OK;
}

template <typename T>
__global__ void to_f32_kernel(const T* src, float* dst, size_t n) {
  size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x;
  if (i < n) dst[i] = float(src[i]);
}

extern "C" int ctd_debug_read_buffer(ctd_handle* h, int32_t buf, float* out, size_t out_elems) {
  NEED_FWD();
  if (buf < 0 || buf >= int(h->bufs.size()) || !out) return ctd_fail(h, CTD_E_INVALID, "bad buffer id");
  const ctd_bufdesc& b = h->bufs[buf];
  const size_t elems = size_t(h->n) * (h->ph / b.down) * (h->pw / b.down) * b.channels;
  if (out_elems < elems) return ctd_fail(h, CTD_E_INVALID, "buffer %d holds %zu elements", buf, elems);
  float* tmp = nullptr;
  CK(cudaMalloc(&tmp, elems * 4));
  if (h->elem == 4) to_f32_kernel<float><<<unsigned((elems + 255) / 256), 256, 0, h->stream>>>(static_cast<float*>(h->d_buf[buf]), tmp, elems);
  else to_f32_kernel<__half><<<unsigned((elems + 255) / 256), 256, 0, h->stream>>>(static_cast<__half*>(h->d_buf[buf]), tmp, elems);
  cudaError_t e = cudaMemcpyAsync(out, tmp, elems * 4, cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(tmp);
  CK(e);
  return CTD_OK;
}

extern "C" int ctd_debug_write_buffer(ctd_handle* h, int32_t buf, const float* in, int32_t n, int32_t ph, int32_t pw) {
  if (!h || !in) return CTD_E_INVALID;
  if (buf < 0 || buf >= int(h->bufs.size())) return ctd_fail(h, CTD_E_INVALID, "bad buffer id");
  if (n < 1 || n > h->cfg.max_batch || ph > h->cfg.max_h || pw > h->cfg.max_w) return ctd_fail(h, CTD_E_CAPACITY, "shape");
  CK(cudaSetDevice(h->cfg.device));
  const ctd_bufdesc& b = h->bufs[buf];
  const size_t elems = size_t(n) * (ph / b.down) * (pw / b.down) * b.channels;
  float* tmp = nullptr;
  CK(cudaMalloc(&tmp, elems * 4));
  cudaError_t e = cudaMemcpyAsync(tmp, in, elems * 4, cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) {
    if (h->elem == 4) from_f32_kernel<float><<<unsigned((elems + 255) / 256), 256, 0, h->stream>>>(tmp, static_cast<float*>(h->d_buf[buf]), elems);
    else from_f32_kernel<__half><<<unsigned((elems + 255) / 256), 256, 0, h->stream>>>(tmp, static_cast<__half*>(h->d_buf[buf]), elems);
    if (h->cfg.precision == CTD_PREC_SPLIT_TC) {
      const size_t npix = elems / b.channels;
      __half* hi = static_cast<__half*>(h->d_buf16[buf]);
      e = split_planes_launch(static_cast<const float*>(h->d_buf[buf]), hi, hi + elems, npix, b.channels, b.channels, h->stream);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  }
  cudaFree(tmp);
  CK(e);
  return CTD_OK;
}

extern "C" int ctd_debug_run_ops(ctd_handle* h, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw, int32_t first_op,
                                 int32_t last_op) {
  if (!h) return CTD_E_INVALID;
  if (first_op < 0 || last_op >= int(h->ops.size()) || first_op > last_op) return ctd_fail(h, CTD_E_INVALID, "bad op range");
  ShapePlan* sp = nullptr;
  if (int rc = find_plan(h, n, ph, pw, &sp)) return rc;
  if (pages) CK(cudaMemcpyAsync(h->d_pages, pages, size_t(n) * ph * pw * 3, cudaMemcpyHostToDevice, h->stream));
  int cnt = 0;
  for (int i = first_op; i <= last_op; ++i)
    if (int rc = run_one_op(h, size_t(i), n, ph, pw, *sp, &cnt)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  h->n = n; h->ph = ph; h->pw = pw;
  h->have_forward = true;
  h->last_launches = cnt;
  return CTD_OK;
}

extern "C" int ctd_debug_postprocess(ctd_handle* h, const float* blks, const float* lines, int32_t n, int32_t ph,
                                     int32_t pw) {
  if (!h || !blks || !lines) return CTD_E_INVALID;
  if (h->cfg.debug_skip_postproc) return ctd_fail(h, CTD_E_INVALID, "ctd_debug_postprocess needs the full pipeline");
  ShapePlan* sp = nullptr;
  if (int rc = find_plan(h, n, ph, pw, &sp)) return rc;
  const size_t hw = size_t(ph) * pw;
  CK(cudaMemcpyAsync(h->d_blks, blks, size_t(n) * rows_per_image(ph, pw) * (5 + h->cfg.nc) * 4, cudaMemcpyHostToDevice,
                     h->stream));
  CK(cudaMemcpyAsync(h->d_lines, lines, size_t(n) * hw * 2 * 4, cudaMemcpyHostToDevice, h->stream));
  // the DB tail's bitmap: the shrink map (channel 0 of each page's lines) > db_thresh, compared in float32
  for (int i = 0; i < n; ++i)
    CK(binarize_launch(h->d_lines + size_t(i) * 2 * hw, hw, h->cfg.db_thresh, h->d_bitmap + size_t(i) * hw, h->stream));
  int cnt = 0;
  if (int rc = launch_nms(h, n, ph, pw, h->stream, &cnt)) return rc;
  if (int rc = launch_db_post(h, n, ph, pw, h->stream, &cnt)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  h->n = n; h->ph = ph; h->pw = pw;
  h->have_forward = true;
  h->last_launches = cnt;
  return CTD_OK;
}

int cc_device(ctd_handle* h, const uint8_t* d_img, int ih, int iw, int stats_cap, int32_t** d_stats, int32_t* n_labels) {
  const size_t px = size_t(ih) * iw;
  // own grow-on-demand scratch (any page size, independent of the net-input workspace; the results of the last
  // forward stay intact): labels | 3 ints/px of CCL scratch (reused for the stats table) | n_labels
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t o_scr = al(px * 4);
  const size_t scr_bytes = al(std::max(px * 12, size_t(stats_cap > 0 ? stats_cap : 0) * 5 * 4));
  const size_t o_nl = o_scr + scr_bytes;
  if (int rc = h->cc_scratch.grow(h, o_nl + 256, h->stream)) return rc;
  uint8_t* base = h->cc_scratch.p;
  int32_t* d_labels = reinterpret_cast<int32_t*>(base);
  int32_t* d_scr = reinterpret_cast<int32_t*>(base + o_scr);
  int32_t* d_nl = reinterpret_cast<int32_t*>(base + o_nl);
  CK(ccl_launch(d_img, 1, ih, iw, d_scr, d_nl, h->stream));
  CK(ccl_number_launch(1, ih, iw, d_scr, d_labels, h->stream));
  if (stats_cap > 0) CK(ccl_stats_launch(d_labels, ih, iw, d_scr, stats_cap, h->stream));   // scratch is free after the numbering
  CK(cudaMemcpyAsync(n_labels, d_nl, 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (d_stats) *d_stats = d_scr;
  return CTD_OK;
}

extern "C" int ctd_connected_components(ctd_handle* h, const uint8_t* img, int32_t ih, int32_t iw, int32_t* labels,
                                        int32_t* stats, int32_t stats_cap, int32_t* n_labels) {
  if (!h || !img || !labels || !n_labels) return CTD_E_INVALID;
  if (ih < 1 || iw < 1 || size_t(ih) * iw > kCclMaxPixels) return ctd_fail(h, CTD_E_SHAPE, "bad image size %dx%d", ih, iw);
  CK(cudaSetDevice(h->cfg.device));
  const size_t px = size_t(ih) * iw;
  if (int rc = h->io_scratch.grow(h, px + 256, h->stream)) return rc;
  CK(cudaMemcpyAsync(h->io_scratch.p, img, px, cudaMemcpyHostToDevice, h->stream));
  int32_t* d_stats = nullptr;
  if (int rc = cc_device(h, h->io_scratch.p, ih, iw, (stats && stats_cap > 0) ? stats_cap : 0, &d_stats, n_labels)) return rc;
  CK(cudaMemcpyAsync(labels, h->cc_scratch.p, px * 4, cudaMemcpyDeviceToHost, h->stream));
  if (stats && stats_cap > 0) CK(cudaMemcpyAsync(stats, d_stats, size_t(stats_cap) * 5 * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_nms(ctd_handle* h, const float* pred, int32_t rows, float conf_thresh, float iou_thresh, float* det,
                       int32_t* det_count) {
  return ctd_nms_dtype(h, pred, rows, CTD_DTYPE_F32, conf_thresh, iou_thresh, det, det_count);
}

extern "C" int ctd_nms_dtype(ctd_handle* h, const void* pred, int32_t rows, int32_t dtype, float conf_thresh,
                             float iou_thresh, float* det, int32_t* det_count) {
  if (!h || !pred || !det || !det_count) return CTD_E_INVALID;
  if (dtype != CTD_DTYPE_F32 && dtype != CTD_DTYPE_F16) return ctd_fail(h, CTD_E_INVALID, "bad dtype %d", dtype);
  const int no = 5 + h->cfg.nc;
  if (rows > rows_per_image(h->cfg.max_h, h->cfg.max_w) * h->cfg.max_batch)
    return ctd_fail(h, CTD_E_CAPACITY, "too many prediction rows");
  CK(cudaSetDevice(h->cfg.device));
  const size_t elems = size_t(rows) * no;
  const int32_t* d_half = nullptr;
  if (dtype == CTD_DTYPE_F16) {
    // the rows widened exactly to float32, as the ingest of ctd_submit_outputs_dtype widens a float16 page, and the
    // page's float16 flag for nms_launch
    std::vector<float> wide(elems);
    const __half* p = static_cast<const __half*>(pred);
    for (size_t i = 0; i < elems; ++i) wide[i] = __half2float(p[i]);
    if (int rc = h->io_scratch.grow(h, 256, h->stream)) return rc;
    const int32_t one = 1;
    CK(cudaMemcpyAsync(h->io_scratch.p, &one, sizeof(one), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_blks, wide.data(), elems * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));   // `one` and `wide` go out of scope here
    d_half = reinterpret_cast<const int32_t*>(h->io_scratch.p);
  } else {
    CK(cudaMemcpyAsync(h->d_blks, pred, elems * 4, cudaMemcpyHostToDevice, h->stream));
  }
  CK(nms_launch(h->d_blks, 1, rows, h->cfg.nc, conf_thresh, iou_thresh, h->nms, h->d_det, h->d_det_count, h->stream,
                d_half));
  CK(cudaMemcpyAsync(det, h->d_det, 300 * 6 * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(det_count, h->d_det_count, 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->have_forward = false;
  return CTD_OK;
}
