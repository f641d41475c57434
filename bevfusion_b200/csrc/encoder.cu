// SparseEncoder as ONE native, sync-free call (replaces the per-conv python loop of
// mmdet3d/models/backbones/sparse_encoder.py:99-132 + spconv/conv.py:114-223 + spconv_ops.h:27-141,260-361).
//
// The reference (and generation 5 of this library) is host paced: every strided conv returns its output
// count to the host (`.item()` / indiceNum.to(kCPU), spconv_ops.h:271) before the next buffer can be
// sized and the next kernel launched.  Here every row count stays on the device:
//   * buffers are sized by CAPS known on the host (level 0: max_voxels; a strided conv can create at most
//     prod(ceil(k/s)) outputs per input and at most one per output site; the caller may pass tighter caps,
//     an overflow flag reports truncation),
//   * kernels take their row count from device memory (grid-stride loops / persistent CTAs),
//   * so the whole encoder -- operand split, 8 rulebooks, 21 convs with folded BN / residual / ReLU
//     epilogues, dense() -- is ~45 launches with no host round trip and can be captured in a CUDA graph.
// Rulebooks depend on the voxel coordinates only; they are built on `rulebook_stream` (when given) and the
// convs wait on one event per rulebook, so they hide behind the convolutions already queued.
//
// Rulebook = offset-major neighbour table nbr[k][row] over the site bitmap of each level's dense grid, built
// by the kernels of rulebook.cu.  Every conv's table is gathered output-side: the rows of the conv's output
// level look their <= K inputs up in the input level's bitmap (no scatter, no -1 fill pass, coalesced writes).
#include <stdlib.h>

#include <algorithm>
#include <new>
#include <vector>

#include "rulebook.cuh"
#include "spconv.cuh"

namespace bevb200 {

__global__ void enc_set_count_kernel(int32_t *dst, int value) { *dst = value; }

// ---- the plan -----------------------------------------------------------------------------------
struct EConv {
  bevb200_encoder_conv_t d;
  int kvol, c_in_eff;
  int level_in, level_out, rulebook;
  bool want_fp32;
  size_t packed_off, scale_off, shift_off;   // offsets into the parameter buffer
  size_t q_off;                              // INT8: [r_out, s_res, s_w[c_out]]
  bool has_scale, has_shift;
};
struct ELevel {
  int shape[3];
  int c_max;           // widest tensor living on this level
};
struct ERulebook {
  int level_q, level_in;   // query (output) level, input level
  int ksize[3], stride[3], pad[3], dil[3];
  int kvol;
};

}  // namespace bevb200

using namespace bevb200;

struct bevb200_encoder {
  int in_channels, c0_eff;
  int precision;                     // BEVB200_PREC_BF16X3 (default), BEVB200_PREC_FP16 or BEVB200_PREC_INT8
  std::vector<EConv> convs;
  std::vector<ELevel> levels;
  std::vector<ERulebook> rulebooks;
  size_t param_bytes;
  std::vector<cudaEvent_t> events;   // [0] fork, [1..] one per rulebook, last: join
  int event_device;
};

namespace bevb200 {

static bool enc_f16(const bevb200_encoder *e) { return e->precision == BEVB200_PREC_FP16; }
static bool enc_i8(const bevb200_encoder *e) { return e->precision == BEVB200_PREC_INT8; }
// bytes per channel of the plan's operand images: BF16x3 split images 4, fp16 images 2 (INT8: enc_level_row_bytes)
static size_t enc_img_bytes(const bevb200_encoder *e) { return enc_f16(e) ? 2 : 4; }

// bytes per row of a level's two images.  INT8: the widest of the level-0 fp16 feature image and the u8 outputs of
// the level's convs; the last conv writes its fp16 image into a buffer of its own (EWs::out16).
static size_t enc_level_row_bytes(const bevb200_encoder *e, size_t l) {
  if (!enc_i8(e)) return (size_t)e->levels[l].c_max * enc_img_bytes(e);
  size_t b = l == 0 ? (size_t)e->c0_eff * 2 : 0;
  for (size_t i = 0; i + 1 < e->convs.size(); ++i)
    if ((size_t)e->convs[i].level_out == l) b = std::max(b, (size_t)e->convs[i].d.c_out);
  return b;
}

// offsets of every conv's packed weights, scale and shift in the parameter buffer (the weight image of the precision).
// INT8: the first conv keeps the fp16 image (it reads the fp16 features), the others take the s8 image; `scale` holds
// the epilogue's factor a[c], and a block [r_out, s_res, s_w[c_out]] follows the shift.
static void enc_param_layout(bevb200_encoder *e) {
  size_t poff = 0;
  for (size_t i = 0; i < e->convs.size(); ++i) {
    EConv &cv = e->convs[i];
    cv.packed_off = poff;
    size_t pk = spconv_v6_packed_bytes(cv.d.c_in, cv.d.c_out, cv.kvol);
    if (enc_f16(e) || (enc_i8(e) && i == 0)) pk = spconv_v6_packed_bytes_f16(cv.d.c_in, cv.d.c_out, cv.kvol);
    else if (enc_i8(e)) pk = spconv_v6_packed_bytes_i8(cv.d.c_in, cv.d.c_out, cv.kvol);
    poff += align_up(pk);
    cv.scale_off = poff; poff += align_up((size_t)cv.d.c_out * 4);
    cv.shift_off = poff; poff += align_up((size_t)cv.d.c_out * 4);
    cv.q_off = poff;
    if (enc_i8(e)) poff += align_up((size_t)(2 + cv.d.c_out) * 4);
  }
  e->param_bytes = poff;
}

static int enc_pack(const bevb200_encoder *e, const EConv &cv, const float *weight, char *params, cudaStream_t st) {
  return enc_f16(e) ? spconv_v6_pack_weights_f16(weight, cv.d.c_in, cv.d.c_out, cv.kvol, params + cv.packed_off, st)
                    : spconv_v6_pack_weights(weight, cv.d.c_in, cv.d.c_out, cv.kvol, params + cv.packed_off, st);
}

static long long level_sites(const ELevel &l, int batch) {
  return (long long)batch * l.shape[0] * l.shape[1] * l.shape[2];
}

// row caps per level: [0] = max_voxels; a strided conv makes <= prod(ceil(k/s)) outputs per input and
// <= 1 per output site; user caps (> 0) may only tighten
static void level_caps(const bevb200_encoder *e, int max_voxels, int batch, const int32_t *user, std::vector<int> *caps) {
  caps->assign(e->levels.size(), 0);
  (*caps)[0] = max_voxels;
  for (const EConv &cv : e->convs) {
    if (cv.level_out == cv.level_in) continue;
    long long fan = 1;
    for (int d = 0; d < 3; ++d) fan *= (cv.d.ksize[d] + cv.d.stride[d] - 1) / cv.d.stride[d];
    long long cap = fan * (*caps)[cv.level_in];
    const long long sites = level_sites(e->levels[cv.level_out], batch);
    if (cap > sites) cap = sites;
    if (user && user[cv.level_out] > 0 && user[cv.level_out] < cap) cap = user[cv.level_out];
    if (cap > 0x7fffff00ll) cap = 0x7fffff00ll;
    (*caps)[cv.level_out] = (int)cap;
  }
}

struct EWs {
  std::vector<SiteBitmap> sites;
  std::vector<int32_t *> indices, counts;
  int32_t *rank2row;
  std::vector<int32_t *> nbr;
  std::vector<uint8_t *> split[2];
  std::vector<float *> f32[2];
  uint8_t *out16;                  // INT8: the last conv's fp16 image, which dense() scatters
  char *zero_begin, *zero_end;
  size_t bytes;
};

// feature_buffers = false: only the rulebook state (the training state keeps its own per-conv rows)
static void enc_layout_into(const bevb200_encoder *e, const std::vector<int> &caps, int batch, Arena &a,
                            bool feature_buffers, EWs *w) {
  const size_t nl = e->levels.size();
  w->sites.resize(nl); w->indices.resize(nl); w->counts.resize(nl);
  // --- region zeroed at the start of every forward: bitmaps, scan state ---
  w->zero_begin = a.base ? a.base + a.off : nullptr;
  for (size_t l = 0; l < nl; ++l) w->sites[l] = take_site_bitmap(a, level_sites(e->levels[l], batch));
  w->zero_end = a.base ? a.base + a.off : nullptr;
  for (size_t l = 0; l < nl; ++l) {
    w->indices[l] = l == 0 ? nullptr : a.take<int32_t>((size_t)caps[l] * 4);
    w->counts[l] = a.take<int32_t>(4);
  }
  w->rank2row = a.take<int32_t>((size_t)caps[0]);
  w->nbr.resize(e->rulebooks.size());
  for (size_t r = 0; r < e->rulebooks.size(); ++r)
    w->nbr[r] = a.take<int32_t>((size_t)e->rulebooks[r].kvol * caps[e->rulebooks[r].level_q]);
  for (int s = 0; s < 2; ++s) {
    w->split[s].assign(nl, nullptr);
    w->f32[s].assign(nl, nullptr);
    if (!feature_buffers) continue;
    for (size_t l = 0; l < nl; ++l) {
      w->split[s][l] = a.take<uint8_t>((size_t)caps[l] * enc_level_row_bytes(e, l));
      // FP16, INT8: dense() scatters the last conv's fp16 image, and residuals are read from images: no fp32 rows
      if (!enc_f16(e) && !enc_i8(e)) w->f32[s][l] = a.take<float>((size_t)caps[l] * e->levels[l].c_max);
    }
  }
  w->out16 = feature_buffers && enc_i8(e) ? a.take<uint8_t>((size_t)caps[nl - 1] * e->convs.back().d.c_out * 2) : nullptr;
  w->bytes = a.off;
}

static size_t enc_layout(const bevb200_encoder *e, const std::vector<int> &caps, int batch, void *ws, size_t ws_bytes,
                         EWs *w) {
  Arena a(ws, ws_bytes);
  enc_layout_into(e, caps, batch, a, true, w);
  return a.off;
}

// Every rulebook of the plan, on stream ss (forked from st with the plan's events when ss != st): the level-0 count,
// the site bitmaps, the output rows of the strided convs and the neighbour tables; status_dev[0] / [1 + l] as in
// bevb200_encoder_forward.  The convs on st wait on events[1 + rulebook] before they read a table.
static int enc_rulebooks(bevb200_encoder *e, const std::vector<int> &caps, int max_voxels, int batch_size,
                         const int32_t *coors, const int32_t *n_voxels_dev, int32_t *status_dev, const EWs &w,
                         cudaStream_t st, cudaStream_t ss) {
  const bool forked = ss != st;
  const size_t nl = e->levels.size(), nr = e->rulebooks.size();
  if (forked) {
    int dev = 0;
    BEVB200_CUDA(cudaGetDevice(&dev));
    if (e->event_device != dev) {
      for (cudaEvent_t ev : e->events) cudaEventDestroy(ev);
      e->events.assign(nr + 2, nullptr);
      for (cudaEvent_t &ev : e->events) BEVB200_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
      e->event_device = dev;
    }
    BEVB200_CUDA(cudaEventRecord(e->events[0], st));       // the coordinates are ready
    BEVB200_CUDA(cudaStreamWaitEvent(ss, e->events[0], 0));
  }
  auto geom_of = [&](const ERulebook &rb) {
    ConvGeom g;
    for (int d = 0; d < 3; ++d) {
      g.in_shape[d] = e->levels[rb.level_in].shape[d];
      g.out_shape[d] = e->levels[rb.level_q].shape[d];
      g.ksize[d] = rb.ksize[d]; g.stride[d] = rb.stride[d]; g.pad[d] = rb.pad[d]; g.dil[d] = rb.dil[d];
    }
    g.batch = batch_size;
    return g;
  };

  BEVB200_CUDA(cudaMemsetAsync(w.zero_begin, 0, (size_t)(w.zero_end - w.zero_begin), ss));
  BEVB200_CUDA(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * (1 + nl), ss));
  // level 0: the caller's rows
  const int32_t *idx0 = coors;
  if (n_voxels_dev) {
    BEVB200_CUDA(cudaMemcpyAsync(w.counts[0], n_voxels_dev, sizeof(int32_t), cudaMemcpyDeviceToDevice, ss));
  } else {
    BEVB200_LAUNCH(enc_set_count_kernel, 1, 1, 0, ss, w.counts[0], max_voxels);
  }
  {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    for (int d = 0; d < 3; ++d) g.in_shape[d] = e->levels[0].shape[d];
    g.batch = batch_size;
    int rc = rb_mark_rows(idx0, caps[0], w.counts[0], g, w.sites[0].cells, ss);
    if (!rc) rc = rb_scan(w.sites[0], ss);
    if (!rc) rc = rb_rank2row(idx0, caps[0], w.counts[0], g, w.sites[0].cells, w.rank2row, ss);
    if (rc) return rc;
  }
  std::vector<char> level_ready(nl, 0);
  level_ready[0] = 1;
  for (size_t r = 0; r < nr; ++r) {
    const ERulebook &rb = e->rulebooks[r];
    const ConvGeom g = geom_of(rb);
    const size_t lq = rb.level_q, li = rb.level_in;
    if (!level_ready[lq]) {
      // a new level: its sites are the outputs of this strided conv
      const int32_t *idx_in = li == 0 ? idx0 : w.indices[li];
      int rc = rb_mark_outputs(idx_in, caps[li], w.counts[li], g, w.sites[lq].cells, ss);
      if (!rc) rc = rb_scan(w.sites[lq], ss);
      if (!rc) rc = rb_count(w.sites[lq].total, caps[lq], w.counts[lq], status_dev, ss);
      if (!rc) rc = rb_out_indices(w.sites[lq], e->levels[lq].shape, caps[lq], w.indices[lq], ss);
      if (rc) return rc;
      level_ready[lq] = 1;
    }
    const int32_t *qidx = lq == 0 ? idx0 : w.indices[lq];
    int rc = rb_gather(qidx, caps[lq], w.counts[lq], g, w.sites[li].cells, li == 0 ? w.rank2row : nullptr, caps[li],
                       w.nbr[r], (long long)caps[lq], ss);
    if (rc) return rc;
    if (forked) BEVB200_CUDA(cudaEventRecord(e->events[1 + r], ss));
  }
  // row counts for the caller: status[1 + l]
  for (size_t l = 0; l < nl; ++l)
    BEVB200_CUDA(cudaMemcpyAsync(status_dev + 1 + l, w.counts[l], sizeof(int32_t), cudaMemcpyDeviceToDevice, ss));
  if (forked) BEVB200_CUDA(cudaEventRecord(e->events[1 + nr], ss));
  return BEVB200_OK;
}

}  // namespace bevb200

extern "C" {

int bevb200_encoder_create(int in_channels, const int32_t *sparse_shape_host, const bevb200_encoder_conv_t *convs,
                           int n_convs, bevb200_encoder_t **out) {
  BEVB200_REQUIRE(out && convs && sparse_shape_host && n_convs > 0 && in_channels > 0, "bad argument");
  bevb200_encoder *e = new (std::nothrow) bevb200_encoder();
  BEVB200_REQUIRE(e != nullptr, "out of host memory");
  e->in_channels = in_channels;
  e->c0_eff = spconv_v6_cin_eff(in_channels);
  e->precision = BEVB200_PREC_BF16X3;
  e->event_device = -1;
  ELevel l0;
  for (int d = 0; d < 3; ++d) l0.shape[d] = sparse_shape_host[d];
  l0.c_max = e->c0_eff;
  e->levels.push_back(l0);
  int level = 0, c_prev = in_channels;
  auto fail = [&](const char *msg) {
    snprintf(g_last_error, sizeof(g_last_error), "bevb200_encoder_create: %s", msg);
    delete e;
    return BEVB200_EINVAL;
  };
  if (e->c0_eff == 0) return fail("in_channels > 128");
  for (int i = 0; i < n_convs; ++i) {
    EConv cv;
    cv.d = convs[i];
    if (cv.d.c_in != c_prev) return fail("conv c_in does not match the previous conv's c_out");
    cv.kvol = cv.d.ksize[0] * cv.d.ksize[1] * cv.d.ksize[2];
    for (int d = 0; d < 3; ++d) {
      if (cv.d.ksize[d] <= 0 || cv.d.dilation[d] <= 0) return fail("bad kernel geometry");
      if (cv.d.subm) {   // spconv_ops.h:74-83: SubM forces stride 1 and padding k/2
        cv.d.stride[d] = 1;
        cv.d.padding[d] = cv.d.ksize[d] / 2;
      }
      if (cv.d.stride[d] <= 0 || cv.d.padding[d] < 0) return fail("bad stride / padding");
    }
    if (!spconv_v6_shape_ok(cv.d.c_in, cv.d.c_out, cv.kvol)) return fail("conv shape has no tensor-core form");
    cv.c_in_eff = spconv_v6_cin_eff(cv.d.c_in);
    if (i > 0 && cv.c_in_eff != cv.d.c_in) return fail("inner channel counts must be multiples of 16");
    if (cv.d.residual_from >= i) return fail("residual_from must name an earlier conv");
    // a level's two split images alternate conv by conv, so conv i - 3's output is overwritten by conv i - 1's
    if (cv.d.residual_from >= 0 && cv.d.residual_from < i - 2)
      return fail("residual_from must name one of the two previous convs");
    cv.level_in = level;
    if (!cv.d.subm) {
      ELevel nl;
      for (int d = 0; d < 3; ++d) {   // ops.py:20-31
        const int num = e->levels[level].shape[d] + 2 * cv.d.padding[d] - cv.d.dilation[d] * (cv.d.ksize[d] - 1) - 1;
        if (num < 0) return fail("conv output shape is empty");
        nl.shape[d] = num / cv.d.stride[d] + 1;
      }
      nl.c_max = cv.d.c_out;
      e->levels.push_back(nl);
      ++level;
    }
    cv.level_out = level;
    if (cv.d.residual_from >= 0) {
      const EConv &src = e->convs[cv.d.residual_from];
      if (src.level_out != cv.level_out || src.d.c_out != cv.d.c_out) return fail("residual shape mismatch");
    }
    e->levels[cv.level_out].c_max = std::max(e->levels[cv.level_out].c_max, cv.d.c_out);
    // rulebook: shared by every conv with the same geometry on the same levels
    cv.rulebook = -1;
    for (size_t r = 0; r < e->rulebooks.size(); ++r) {
      const ERulebook &rb = e->rulebooks[r];
      bool same = rb.level_q == cv.level_out && rb.level_in == cv.level_in;
      for (int d = 0; d < 3 && same; ++d)
        same = rb.ksize[d] == cv.d.ksize[d] && rb.stride[d] == cv.d.stride[d] && rb.pad[d] == cv.d.padding[d] &&
               rb.dil[d] == cv.d.dilation[d];
      if (same) cv.rulebook = (int)r;
    }
    if (cv.rulebook < 0) {
      ERulebook rb;
      rb.level_q = cv.level_out;
      rb.level_in = cv.level_in;
      for (int d = 0; d < 3; ++d) {
        rb.ksize[d] = cv.d.ksize[d]; rb.stride[d] = cv.d.stride[d]; rb.pad[d] = cv.d.padding[d]; rb.dil[d] = cv.d.dilation[d];
      }
      rb.kvol = cv.kvol;
      cv.rulebook = (int)e->rulebooks.size();
      e->rulebooks.push_back(rb);
    }
    cv.want_fp32 = i == n_convs - 1;
    cv.has_scale = cv.has_shift = false;
    e->convs.push_back(cv);
    c_prev = cv.d.c_out;
  }
  // A residual is read from the source conv's SPLIT image -- hi + lo is the value to 2^-17 -- so only the last conv,
  // whose rows dense() scatters, writes fp32 rows; BEVB200_ENCODER_F32_RESIDUAL=1 restores the fp32 residual copies.
  static const bool f32_residual = [] { const char *v = getenv("BEVB200_ENCODER_F32_RESIDUAL"); return v && atoi(v) != 0; }();
  for (EConv &cv : e->convs)
    if (f32_residual && cv.d.residual_from >= 0) e->convs[cv.d.residual_from].want_fp32 = true;
  enc_param_layout(e);
  *out = e;
  return BEVB200_OK;
}

void bevb200_encoder_destroy(bevb200_encoder_t *e) {
  if (!e) return;
  for (cudaEvent_t ev : e->events) cudaEventDestroy(ev);
  delete e;
}

int bevb200_encoder_set_precision(bevb200_encoder_t *e, int precision) {
  BEVB200_REQUIRE(e, "null plan");
  BEVB200_REQUIRE(precision == BEVB200_PREC_BF16X3 || precision == BEVB200_PREC_FP16 || precision == BEVB200_PREC_INT8,
                  "an encoder plan runs BEVB200_PREC_BF16X3, BEVB200_PREC_FP16 or BEVB200_PREC_INT8");
  if (precision == BEVB200_PREC_INT8)   // every stored activation is >= 0: the u8 images
    for (const EConv &cv : e->convs) BEVB200_REQUIRE(cv.d.relu, "an INT8 plan needs a ReLU after every conv");
  e->precision = precision;
  enc_param_layout(e);
  return BEVB200_OK;
}

int bevb200_encoder_precision(const bevb200_encoder_t *e) { return e ? e->precision : BEVB200_EINVAL; }

size_t bevb200_encoder_param_bytes(const bevb200_encoder_t *e) { return e ? e->param_bytes : 0; }

int bevb200_encoder_num_levels(const bevb200_encoder_t *e) { return e ? (int)e->levels.size() : 0; }

int bevb200_encoder_output_shape(const bevb200_encoder_t *e, int32_t *shape_out, int32_t *channels_out) {
  BEVB200_REQUIRE(e && shape_out && channels_out, "null argument");
  for (int d = 0; d < 3; ++d) shape_out[d] = e->levels.back().shape[d];
  *channels_out = e->convs.back().d.c_out;
  return BEVB200_OK;
}

int bevb200_encoder_set_conv(bevb200_encoder_t *e, int conv, const float *weight, const float *scale,
                             const float *shift, void *params, size_t params_bytes, void *stream) {
  BEVB200_REQUIRE(e && conv >= 0 && conv < (int)e->convs.size(), "bad conv index");
  BEVB200_REQUIRE(!enc_i8(e), "an INT8 plan packs its convs with bevb200_encoder_set_conv_int8");
  BEVB200_REQUIRE(weight && params && params_bytes >= e->param_bytes, "null argument / parameter buffer too small");
  EConv &cv = e->convs[conv];
  cudaStream_t st = (cudaStream_t)stream;
  char *base = (char *)params;
  int rc = enc_pack(e, cv, weight, base, st);
  if (rc) return rc;
  cv.has_scale = scale != nullptr;
  cv.has_shift = shift != nullptr;
  if (scale)
    BEVB200_CUDA(cudaMemcpyAsync(base + cv.scale_off, scale, (size_t)cv.d.c_out * 4, cudaMemcpyDeviceToDevice, st));
  if (shift)
    BEVB200_CUDA(cudaMemcpyAsync(base + cv.shift_off, shift, (size_t)cv.d.c_out * 4, cudaMemcpyDeviceToDevice, st));
  return BEVB200_OK;
}

}  // extern "C"

// INT8 epilogue parameters of one conv: a[c] = bn_scale[c] (the first conv) or fl(fl(s_in * s_w[c]) * bn_scale[c])
// (bn_scale = 1 when absent), the shift (0 when absent), r_out = fl(1 / s_out) and s_res
__global__ void enc_i8_epilogue_kernel(const float *__restrict__ bn_scale, const float *__restrict__ shift, int c_out,
                                       int first, float s_in, float s_out, float s_res, float *__restrict__ a,
                                       float *__restrict__ shift_out, float *__restrict__ q) {
  const float *s_w = q + 2;
  for (int c = threadIdx.x; c < c_out; c += blockDim.x) {
    const float sc = bn_scale ? bn_scale[c] : 1.f;
    a[c] = first ? sc : __fmul_rn(__fmul_rn(s_in, s_w[c]), sc);
    shift_out[c] = shift ? shift[c] : 0.f;
  }
  if (threadIdx.x == 0) {
    q[0] = __fdiv_rn(1.f, s_out);
    q[1] = s_res;
  }
}

extern "C" {

int bevb200_encoder_set_conv_int8(bevb200_encoder_t *e, int conv, const float *weight, const float *scale,
                                  const float *shift, float s_in, float s_out, float s_res, void *params,
                                  size_t params_bytes, void *stream) {
  BEVB200_REQUIRE(e && conv >= 0 && conv < (int)e->convs.size(), "bad conv index");
  BEVB200_REQUIRE(enc_i8(e), "bevb200_encoder_set_conv_int8 needs a plan set to BEVB200_PREC_INT8");
  BEVB200_REQUIRE(weight && params && params_bytes >= e->param_bytes, "null argument / parameter buffer too small");
  EConv &cv = e->convs[conv];
  auto scale_ok = [](float s) { return s > 0.f && s <= 3.4e38f; };
  BEVB200_REQUIRE(scale_ok(s_out) && (conv == 0 || scale_ok(s_in)) && (cv.d.residual_from < 0 || scale_ok(s_res)),
                  "activation scales must be finite and > 0");
  cudaStream_t st = (cudaStream_t)stream;
  char *base = (char *)params;
  float *q = (float *)(base + cv.q_off);
  int rc = conv == 0 ? spconv_v6_pack_weights_f16(weight, cv.d.c_in, cv.d.c_out, cv.kvol, base + cv.packed_off, st)
                     : spconv_v6_pack_weights_i8(weight, cv.d.c_in, cv.d.c_out, cv.kvol, q + 2, base + cv.packed_off, st);
  if (rc) return rc;
  BEVB200_LAUNCH(enc_i8_epilogue_kernel, 1, 128, 0, st, scale, shift, cv.d.c_out, conv == 0 ? 1 : 0, s_in, s_out,
                 cv.d.residual_from >= 0 ? s_res : 0.f, (float *)(base + cv.scale_off), (float *)(base + cv.shift_off), q);
  cv.has_scale = cv.has_shift = true;
  return BEVB200_OK;
}

int bevb200_encoder_level_caps(const bevb200_encoder_t *e, int max_voxels, int batch_size, const int32_t *user_caps,
                               int32_t *caps_out) {
  BEVB200_REQUIRE(e && caps_out && max_voxels > 0 && batch_size > 0, "bad argument");
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  for (size_t l = 0; l < caps.size(); ++l) caps_out[l] = caps[l];
  return BEVB200_OK;
}

size_t bevb200_encoder_workspace_bytes(const bevb200_encoder_t *e, int max_voxels, int batch_size,
                                       const int32_t *user_caps) {
  if (!e || max_voxels <= 0 || batch_size <= 0) return 0;
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  EWs w;
  return enc_layout(e, caps, batch_size, nullptr, 0, &w);
}

}  // extern "C"

// bevb200_encoder_forward(_f16): voxel_features and dense_out are fp32 (BF16x3 plan) or fp16 (FP16 and INT8 plans)
static int enc_forward(bevb200_encoder_t *e, bool f16, const void *params, const void *voxel_features,
                       const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev, int batch_size,
                       const int32_t *user_caps, void *dense_out, long long out_batch_stride, int32_t *status_dev,
                       void *workspace, size_t workspace_bytes, void *stream, void *rulebook_stream) {
  // the precision first: a call of the wrong family is refused before any other argument is looked at
  BEVB200_REQUIRE(e, "null plan");
  BEVB200_REQUIRE((enc_f16(e) || enc_i8(e)) == f16,
                  f16 ? "the _f16 calls need a plan set to BEVB200_PREC_FP16 or BEVB200_PREC_INT8"
                      : "fp16 and INT8 plans run the _f16 calls");
  const bool i8 = enc_i8(e);
  BEVB200_REQUIRE(e && params && dense_out && status_dev && max_voxels > 0 && batch_size > 0, "bad argument");
  BEVB200_REQUIRE(voxel_features && coors, "null input");
  cudaStream_t st = (cudaStream_t)stream, ss = rulebook_stream ? (cudaStream_t)rulebook_stream : st;
  const bool forked = ss != st;
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  EWs w;
  const size_t need = enc_layout(e, caps, batch_size, workspace, workspace_bytes, &w);
  if (workspace == nullptr || workspace_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "encoder_forward: workspace too small (%zu < %zu)", workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  const size_t nl = e->levels.size(), nr = e->rulebooks.size();
  const char *pbase = (const char *)params;
  const int32_t *idx0 = coors;
  // ------------------------------ rulebooks (stream ss) ------------------------------------
  int rc = enc_rulebooks(e, caps, max_voxels, batch_size, coors, n_voxels_dev, status_dev, w, st, ss);
  if (rc) return rc;

  // ------------------------------ features (stream st) -------------------------------------
  rc = f16 ? spconv_v6_f16_rows((const __half *)voxel_features, caps[0], n_voxels_dev, e->in_channels, e->c0_eff,
                                 w.split[0][0], st)
           : spconv_v6_split_rows((const float *)voxel_features, caps[0], n_voxels_dev, e->in_channels, e->c0_eff,
                                  w.split[0][0], st);
  if (rc) return rc;
  std::vector<int> split_turn(nl, 0), f32_turn(nl, 0);
  split_turn[0] = 1;
  const uint8_t *cur_split = w.split[0][0];
  std::vector<const float *> f32_of(e->convs.size(), nullptr);
  std::vector<const uint8_t *> split_of(e->convs.size(), nullptr);
  std::vector<char> rb_waited(nr, 0);
  const float *last_f32 = nullptr;
  for (size_t i = 0; i < e->convs.size(); ++i) {
    const EConv &cv = e->convs[i];
    if (forked && !rb_waited[cv.rulebook]) {
      BEVB200_CUDA(cudaStreamWaitEvent(st, e->events[1 + cv.rulebook], 0));
      rb_waited[cv.rulebook] = 1;
    }
    const size_t lo = cv.level_out;
    const bool last = i + 1 == e->convs.size();
    uint8_t *osplit = nullptr;
    if (i8 && last) {
      osplit = w.out16;
    } else if (!last || f16) {   // FP16: the last conv's image is what dense() scatters
      osplit = w.split[split_turn[lo]][lo];
      split_turn[lo] ^= 1;
    }
    float *of32 = nullptr;
    if (cv.want_fp32 && !f16) {
      of32 = w.f32[f32_turn[lo]][lo];
      f32_turn[lo] ^= 1;
      f32_of[i] = of32;
    }
    // residual: the source conv's fp32 rows if it wrote them, else its split image (which may be the buffer this conv
    // writes: the two split buffers of a level alternate and a block's input is two convs back -- safe, see spconv_v6.cu)
    const float *res = cv.d.residual_from >= 0 ? f32_of[cv.d.residual_from] : nullptr;
    const uint8_t *res_split = (cv.d.residual_from >= 0 && res == nullptr) ? split_of[cv.d.residual_from] : nullptr;
    BEVB200_REQUIRE(cv.d.residual_from < 0 || res || res_split, "residual source has no rows");
    if (i8)
      rc = spconv_v6_forward_i8(cur_split, i == 0, pbase + cv.packed_off, w.nbr[cv.rulebook], (long long)caps[lo],
                                caps[cv.level_in], caps[lo], w.counts[lo], cv.c_in_eff, cv.d.c_out, cv.kvol,
                                (const float *)(pbase + cv.scale_off), (const float *)(pbase + cv.shift_off),
                                (const float *)(pbase + cv.q_off), res_split, cv.d.relu, last, osplit, st);
    else
      rc = (f16 ? spconv_v6_forward_f16 : spconv_v6_forward)(
        cur_split, pbase + cv.packed_off, w.nbr[cv.rulebook], (long long)caps[lo], caps[cv.level_in], caps[lo],
        w.counts[lo], cv.c_in_eff, cv.d.c_out, cv.kvol, cv.has_scale ? (const float *)(pbase + cv.scale_off) : nullptr,
        cv.has_shift ? (const float *)(pbase + cv.shift_off) : nullptr, res, res_split, cv.d.relu, of32, osplit, st);
    if (rc) return rc;
    split_of[i] = osplit;
    cur_split = osplit;
    last_f32 = of32;
  }
  // dense(): [B, C*Z, X, Y]
  const size_t ll = nl - 1;
  const int32_t *lidx = w.indices[ll] ? w.indices[ll] : idx0;
  rc = f16 ? sparse_to_dense((const __half *)cur_split, lidx, caps[ll], w.counts[ll], e->convs.back().d.c_out,
                             batch_size, e->levels[ll].shape, 1, out_batch_stride, (__half *)dense_out, st)
           : sparse_to_dense(last_f32, lidx, caps[ll], w.counts[ll], e->convs.back().d.c_out, batch_size,
                             e->levels[ll].shape, 1, out_batch_stride, (float *)dense_out, st);
  if (rc) return rc;
  if (forked) BEVB200_CUDA(cudaStreamWaitEvent(st, e->events[1 + nr], 0));   // join (also what a graph capture needs)
  return BEVB200_OK;
}

extern "C" {

int bevb200_encoder_forward(bevb200_encoder_t *e, const void *params, const float *voxel_features,
                            const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev, int batch_size,
                            const int32_t *user_caps, float *dense_out, long long out_batch_stride,
                            int32_t *status_dev, void *workspace, size_t workspace_bytes, void *stream,
                            void *rulebook_stream) {
  return enc_forward(e, false, params, voxel_features, coors, max_voxels, n_voxels_dev, batch_size, user_caps,
                     dense_out, out_batch_stride, status_dev, workspace, workspace_bytes, stream, rulebook_stream);
}

int bevb200_encoder_forward_f16(bevb200_encoder_t *e, const void *params, const void *voxel_features,
                                const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev, int batch_size,
                                const int32_t *user_caps, void *dense_out, long long out_batch_stride,
                                int32_t *status_dev, void *workspace, size_t workspace_bytes, void *stream,
                                void *rulebook_stream) {
  return enc_forward(e, true, params, voxel_features, coors, max_voxels, n_voxels_dev, batch_size, user_caps,
                     dense_out, out_batch_stride, status_dev, workspace, workspace_bytes, stream, rulebook_stream);
}

}  // extern "C"

// ================================== training ====================================================
// forward_train: rulebooks as above, then per conv
//   conv (no epilogue) -> z fp32 | stats partials (double, fixed 2048-row chunks) | stats reduce (mean, invstd,
//   scale = gamma invstd, shift = beta - mean scale; running statistics) | apply y = relu(z scale + shift [+ y_res])
//   into the split image the next conv gathers (and the backward reads again).
// backward, in reverse conv order, on the same tables:
//   ReLU mask + BN sums (double partials of g and g x^, fixed order) | reduce (dgamma, dbeta) | dz |
//   filter gradient on the saved input image (spconv_wgrad_tc_split) | input gradient = the forward kernel on W^T:
//   SubM: the forward table with mirrored offsets, strided: a transposed table; a block's identity gradient rides in
//   the residual epilogue of the input gradient of the conv that reads the identity.
// FP16 plans (BEVB200_PREC_FP16) run the same sequence with fp16 rows: the conv writes z16 = fp16(acc), the statistics
// and the BN backward read z16, the apply writes the fp16 image y16 that the next conv gathers, dense() scatters the
// last y16, and dz is rounded once to an fp16 image that both the filter gradient and the input gradient read.
#include "tc_ptx.cuh"

namespace bevb200 {

constexpr int kStatRows = 2048;   // rows per partial of the BN sums
constexpr int kStatThreads = 256;

static int stat_chunks(int cap) { return cap > 0 ? (cap + kStatRows - 1) / kStatRows : 1; }

__device__ __forceinline__ int enc_rows(const int32_t *n_dev, int cap) { return min(max(__ldg(n_dev), 0), cap); }

__device__ __forceinline__ float ld_f(const float *p) { return *p; }
__device__ __forceinline__ float ld_f(const __half *p) { return __half2float(*p); }
__device__ __forceinline__ void st_f(float *p, float v) { *p = v; }
__device__ __forceinline__ void st_f(__half *p, float v) { *p = __float2half_rn(v); }
// rows of the BF16x3 / FP16 forms: pre-BN rows z and dz are fp32 / fp16
template <bool F16>
using enc_row_t = typename std::conditional<F16, __half, float>::type;

// value of channel ch of row r of a split image (F16: an fp16 image) with c channels per row
template <bool F16 = false>
__device__ __forceinline__ float split_value(const uint8_t *img, long long r, int c, int ch) {
  if (F16) return __half2float(reinterpret_cast<const __half *>(img)[r * c + ch]);
  const uint8_t *p = img + r * (c * 4) + (ch >> 4) * 64 + (ch & 15) * 2;
  const uint32_t h = *reinterpret_cast<const uint16_t *>(p), l = *reinterpret_cast<const uint16_t *>(p + 32);
  return __uint_as_float(h << 16) + __uint_as_float(l << 16);
}

// thread (group g, channel ch) of a 256-thread block over c channels: c <= 128, so >= 2 groups
#define STAT_THREAD(c)                                 \
  const int groups = kStatThreads / (c);               \
  const int ch = threadIdx.x % (c), grp = threadIdx.x / (c)

// per-channel sums of v and v^2 (double) over the rows of one chunk; the groups add in ascending order
template <typename T>
__global__ void __launch_bounds__(kStatThreads)
    bn_stats_partial_kernel(const T *__restrict__ z, const int32_t *__restrict__ n_dev, int cap, int c,
                            double *__restrict__ partial) {
  __shared__ double sh[2][kStatThreads];
  STAT_THREAD(c);
  const int n = enc_rows(n_dev, cap);
  const int r0 = blockIdx.x * kStatRows, r1 = min(n, r0 + kStatRows);
  if (r0 >= n) return;                           // chunks past the count are never read
  double s = 0.0, ss = 0.0;
  if (grp < groups)
    for (int r = r0 + grp; r < r1; r += groups) {
      const double v = ld_f(z + (long long)r * c + ch);
      s += v;
      ss += v * v;
    }
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = ss;
  __syncthreads();
  if (threadIdx.x < c) {
    for (int q = 1; q < groups; ++q) { s += sh[0][q * c + ch]; ss += sh[1][q * c + ch]; }
    partial[(long long)blockIdx.x * 2 * c + ch] = s;
    partial[(long long)blockIdx.x * 2 * c + c + ch] = ss;
  }
}

// sums of the partials of the chunks that hold rows, in a fixed order; thread ch < c returns its channel's two sums
__device__ __forceinline__ void stat_sums(const double *__restrict__ partial, int n, int c, double *sh, double &s,
                                          double &ss) {
  STAT_THREAD(c);
  const int chunks = (n + kStatRows - 1) / kStatRows;
  s = 0.0; ss = 0.0;
  if (grp < groups)
    for (int k = grp; k < chunks; k += groups) {
      s += partial[(long long)k * 2 * c + ch];
      ss += partial[(long long)k * 2 * c + c + ch];
    }
  sh[threadIdx.x] = s;
  sh[kStatThreads + threadIdx.x] = ss;
  __syncthreads();
  if (threadIdx.x < c)
    for (int q = 1; q < groups; ++q) { s += sh[q * c + ch]; ss += sh[kStatThreads + q * c + ch]; }
}

// batch statistics -> stat [mean | invstd | scale | shift] and the running statistics (torch's BatchNorm1d, train)
__global__ void __launch_bounds__(kStatThreads)
    bn_stats_reduce_kernel(const double *__restrict__ partial, const int32_t *__restrict__ n_dev, int cap, int c,
                           bevb200_encoder_bn_t bn, float *__restrict__ stat, int32_t *__restrict__ status) {
  __shared__ double sh[2 * kStatThreads];
  const int n = enc_rows(n_dev, cap);
  double s, ss;
  stat_sums(partial, n, c, sh, s, ss);
  const int ch = threadIdx.x;
  if (ch >= c) return;
  const double mean = n > 0 ? s / n : 0.0;
  const double var = n > 0 ? fmax(ss / n - mean * mean, 0.0) : 0.0;    // biased: the normalisation's
  const double invstd = 1.0 / sqrt(var + (double)bn.eps);
  const double scale = (double)bn.weight[ch] * invstd;
  stat[ch] = (float)mean;
  stat[c + ch] = (float)invstd;
  stat[2 * c + ch] = (float)scale;
  stat[3 * c + ch] = (float)((double)bn.bias[ch] - mean * scale);
  if (n >= 2) {
    const double m = bn.momentum;
    bn.running_mean[ch] = (float)((1.0 - m) * bn.running_mean[ch] + m * mean);
    bn.running_var[ch] = (float)((1.0 - m) * bn.running_var[ch] + m * var * n / (n - 1.0));
    if (ch == 0 && bn.num_batches_tracked) *bn.num_batches_tracked += 1;
  } else if (ch == 0) {
    atomicOr(status, BEVB200_ENCODER_FEW_ROWS);
  }
}

// y = relu(z scale + shift [+ residual image]) -> split image (and fp32 rows); one thread per (row, 8 channels).
// F16: z, the residual and y are fp16 images; y is rounded once.
template <bool F16>
__global__ void bn_apply_kernel(const enc_row_t<F16> *__restrict__ z, const float *__restrict__ stat,
                                const uint8_t *__restrict__ res_split, const int32_t *__restrict__ n_dev, int cap,
                                int c, int relu, uint8_t *__restrict__ ysplit, float *__restrict__ yf32) {
  const int n = enc_rows(n_dev, cap);
  const int per_row = c >> 3;
  const long long total = (long long)n * per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(t % per_row), c0 = 8 * j;
    const long long r = t / per_row;
    float y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = ld_f(z + r * c + c0 + e);
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = y[e] * __ldg(stat + 2 * c + c0 + e) + __ldg(stat + 3 * c + c0 + e);
    if (res_split) {
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] += split_value<F16>(res_split, r, c, c0 + e);
    }
    if (relu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = fmaxf(y[e], 0.f);
    }
    if (yf32) {
      *reinterpret_cast<float4 *>(yf32 + r * c + c0) = make_float4(y[0], y[1], y[2], y[3]);
      *reinterpret_cast<float4 *>(yf32 + r * c + c0 + 4) = make_float4(y[4], y[5], y[6], y[7]);
    }
    if constexpr (F16) {
      __half *dst = reinterpret_cast<__half *>(ysplit) + r * c + c0;
#pragma unroll
      for (int e = 0; e < 8; ++e) dst[e] = __float2half_rn(y[e]);
    } else {
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int e = 0; e < 8; e += 2) split_pair(y[e], y[e + 1], hi[e / 2], lo[e / 2]);
      uint8_t *dst = ysplit + r * (c * 4) + (j >> 1) * 64 + (j & 1) * 16;
      *reinterpret_cast<uint4 *>(dst) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<uint4 *>(dst + 32) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
  }
}

// rows of the last level from the dense gradient (the inverse of sparse_to_dense with z_major)
template <typename T>
__global__ void dense_gather_kernel(const T *__restrict__ dense, const int32_t *__restrict__ idx,
                                    const int32_t *__restrict__ n_dev, int cap, int c, int batch, int X, int Y, int Z,
                                    long long out_batch_stride, float *__restrict__ rows) {
  const int n = enc_rows(n_dev, cap);
  const long long total = (long long)n * c, plane = (long long)X * Y * Z;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(t % n), ch = (int)(t / n);
    const int4 p = *reinterpret_cast<const int4 *>(idx + 4ll * i);
    float v = 0.f;
    if ((unsigned)p.x < (unsigned)batch && (unsigned)p.y < (unsigned)X && (unsigned)p.z < (unsigned)Y &&
        (unsigned)p.w < (unsigned)Z)
      v = ld_f(dense + p.x * out_batch_stride + ch * plane + ((long long)p.w * X + p.y) * Y + p.z);
    rows[(long long)i * c + ch] = v;
  }
}

// ReLU mask applied to g in place, then per-channel sums of g and g x^ (x^ = (z - mean) invstd) per chunk
template <bool F16>
__global__ void __launch_bounds__(kStatThreads)
    bn_bwd_partial_kernel(float *__restrict__ g, const uint8_t *__restrict__ ysplit, const float *__restrict__ yf32,
                          int relu, const enc_row_t<F16> *__restrict__ z, const float *__restrict__ stat,
                          const int32_t *__restrict__ n_dev, int cap, int c, double *__restrict__ partial) {
  __shared__ double sh[2][kStatThreads];
  STAT_THREAD(c);
  const int n = enc_rows(n_dev, cap);
  const int r0 = blockIdx.x * kStatRows, r1 = min(n, r0 + kStatRows);
  if (r0 >= n) return;
  double s = 0.0, sx = 0.0;
  if (grp < groups) {
    const float mean = stat[ch], invstd = stat[c + ch];
    for (int r = r0 + grp; r < r1; r += groups) {
      const long long e = (long long)r * c + ch;
      float gv = g[e];
      if (relu) {
        const float y = yf32 ? yf32[e] : split_value<F16>(ysplit, r, c, ch);
        if (!(y > 0.f)) gv = 0.f;
        g[e] = gv;
      }
      s += gv;
      sx += (double)gv * (double)((ld_f(z + e) - mean) * invstd);
    }
  }
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = sx;
  __syncthreads();
  if (threadIdx.x < c) {
    for (int q = 1; q < groups; ++q) { s += sh[0][q * c + ch]; sx += sh[1][q * c + ch]; }
    partial[(long long)blockIdx.x * 2 * c + ch] = s;
    partial[(long long)blockIdx.x * 2 * c + c + ch] = sx;
  }
}

// dbeta = sum g, dgamma = sum g x^; coef = [sum g / n | sum g x^ / n]
__global__ void __launch_bounds__(kStatThreads)
    bn_bwd_reduce_kernel(const double *__restrict__ partial, const int32_t *__restrict__ n_dev, int cap, int c,
                         float *__restrict__ dgamma, float *__restrict__ dbeta, float *__restrict__ coef) {
  __shared__ double sh[2 * kStatThreads];
  const int n = enc_rows(n_dev, cap);
  double s, sx;
  stat_sums(partial, n, c, sh, s, sx);
  const int ch = threadIdx.x;
  if (ch >= c) return;
  dbeta[ch] = (float)s;
  dgamma[ch] = (float)sx;
  coef[ch] = n > 0 ? (float)(s / n) : 0.f;
  coef[c + ch] = n > 0 ? (float)(sx / n) : 0.f;
}

// dz = gamma invstd (g - mean(g) - x^ mean(g x^)); F16: z16 in, dz rounded once to fp16
template <bool F16>
__global__ void bn_bwd_apply_kernel(const float *__restrict__ g, const enc_row_t<F16> *__restrict__ z,
                                    const float *__restrict__ stat, const float *__restrict__ coef,
                                    const int32_t *__restrict__ n_dev, int cap, int c, enc_row_t<F16> *__restrict__ dz) {
  const int n = enc_rows(n_dev, cap);
  const long long total = (long long)n * c;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(t % c);
    const float xh = (ld_f(z + t) - __ldg(stat + ch)) * __ldg(stat + c + ch);
    st_f(dz + t, __ldg(stat + 2 * c + ch) * (g[t] - __ldg(coef + ch) - xh * __ldg(coef + c + ch)));
  }
}

// wt[k][co][ci] = w[mirror ? K-1-k : k][ci][co], ci zero padded to ci_pad
__global__ void enc_weight_t_kernel(const float *__restrict__ w, int kvol, int c_in, int c_out, int ci_pad, int mirror,
                                    float *__restrict__ wt) {
  const long long total = (long long)kvol * c_out * ci_pad;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(t % ci_pad), co = (int)((t / ci_pad) % c_out), k = (int)(t / ((long long)ci_pad * c_out));
    const int ks = mirror ? kvol - 1 - k : k;
    wt[t] = ci < c_in ? w[((long long)ks * c_in + ci) * c_out + co] : 0.f;
  }
}

// nbr_t[k][j] = -1 for the valid input rows j, then nbr_t[k][nbr[k][o]] = o for the valid output rows o
__global__ void enc_nbr_t_fill_kernel(const int32_t *__restrict__ n_in_dev, int cap_in, int kvol,
                                      int32_t *__restrict__ nbr_t) {
  const int n = enc_rows(n_in_dev, cap_in);
  const long long total = (long long)kvol * n;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x)
    nbr_t[(t / n) * cap_in + t % n] = -1;
}
__global__ void enc_nbr_t_scatter_kernel(const int32_t *__restrict__ nbr, const int32_t *__restrict__ n_out_dev,
                                         int cap_out, const int32_t *__restrict__ n_in_dev, int cap_in, int kvol,
                                         int32_t *__restrict__ nbr_t) {
  const int n = enc_rows(n_out_dev, cap_out), n_in = enc_rows(n_in_dev, cap_in);
  const long long total = (long long)kvol * n;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const long long k = t / n;
    const int o = (int)(t % n);
    const int j = nbr[k * cap_out + o];
    if (j >= 0 && j < n_in) nbr_t[k * cap_in + j] = o;   // one writer per (k, j)
  }
}

// split image rows of c_src channels -> rows of c_dst >= c_src channels (zero padded), for the filter gradient
__global__ void enc_widen_image_kernel(const uint8_t *__restrict__ src, int c_src, int c_dst,
                                       const int32_t *__restrict__ n_dev, int cap, uint8_t *__restrict__ dst) {
  const int n = enc_rows(n_dev, cap);
  const int per_row = c_dst / 4;   // 16-byte chunks
  const long long total = (long long)n * per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const long long r = t / per_row;
    const int q = (int)(t % per_row);
    const uint4 v = q < c_src / 4 ? *reinterpret_cast<const uint4 *>(src + r * c_src * 4 + 16 * q) : make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(dst + r * c_dst * 4 + 16 * q) = v;
  }
}

// input gradient rows [cap, c_eff] -> grad_voxel_features [rows, c_in]: the valid rows narrowed, the rest zero
template <typename T>
__global__ void enc_narrow_grad_kernel(const float *__restrict__ src, int c_eff, const int32_t *__restrict__ n_dev,
                                       int cap, int rows, int c_in, T *__restrict__ dst) {
  const int n = enc_rows(n_dev, cap);
  const long long total = (long long)rows * c_in;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const long long r = t / c_in;
    st_f(dst + t, r < n ? src[r * c_eff + t % c_in] : 0.f);
  }
}

// ---- state and workspace layouts ----
struct ETrain {
  EWs w;
  char *params;
  uint8_t *in_split;              // level-0 split image (FP16: fp16 image) of the voxel features
  std::vector<void *> z;          // pre-BN rows per conv: fp32 (FP16: z16 = fp16(acc))
  std::vector<uint8_t *> y;       // split image (FP16: fp16 image) of every conv's output
  std::vector<float *> stat;      // per conv [mean | invstd | scale | shift][c_out]
  float *y_last;                  // BF16x3: fp32 rows of the last conv (dense() and its ReLU mask)
  double *partial;
};

static size_t train_layout(const bevb200_encoder *e, const std::vector<int> &caps, int batch, void *base,
                           size_t bytes, ETrain *t) {
  Arena a(base, bytes);
  enc_layout_into(e, caps, batch, a, false, &t->w);
  t->params = a.take<char>(e->param_bytes);
  const size_t ib = enc_img_bytes(e);
  t->in_split = a.take<uint8_t>((size_t)caps[0] * e->c0_eff * ib);
  const size_t n = e->convs.size();
  t->z.resize(n); t->y.resize(n); t->stat.resize(n);
  size_t part = 0;
  for (size_t i = 0; i < n; ++i) {
    const EConv &cv = e->convs[i];
    const size_t cap = caps[cv.level_out];
    t->z[i] = a.take<uint8_t>(cap * cv.d.c_out * (enc_f16(e) ? 2 : 4));
    t->y[i] = a.take<uint8_t>(cap * cv.d.c_out * ib);
    t->stat[i] = a.take<float>(4 * (size_t)cv.d.c_out);
    part = std::max(part, (size_t)stat_chunks(caps[cv.level_out]) * 2 * cv.d.c_out);
  }
  t->y_last = enc_f16(e) ? nullptr : a.take<float>((size_t)caps.back() * e->convs.back().d.c_out);
  t->partial = a.take<double>(part);
  return a.off;
}

struct EBwd {
  std::vector<float *> d[2];      // per level: two gradient row buffers
  std::vector<void *> dz;         // per level: the dz rows (FP16: the fp16 image of dz)
  int32_t *nbr_t;
  float *wt, *coef, *din0;
  char *packed, *wg;
  uint8_t *fwide, *g16;
  double *partial;
};

static size_t bwd_layout(const bevb200_encoder *e, const std::vector<int> &caps, void *base, size_t bytes, EBwd *b) {
  Arena a(base, bytes);
  const size_t nl = e->levels.size();
  for (int s = 0; s < 2; ++s) b->d[s].resize(nl);
  b->dz.resize(nl);
  for (size_t l = 0; l < nl; ++l) {
    const size_t n = (size_t)caps[l] * e->levels[l].c_max;
    b->d[0][l] = a.take<float>(n);
    b->d[1][l] = a.take<float>(n);
    b->dz[l] = a.take<uint8_t>(n * (enc_f16(e) ? 2 : 4));
  }
  size_t nbrt = 0, wt = 0, pk = 0, wg = 0, fw = 0, g16 = 0, part = 0, cmax = 0;
  for (const EConv &cv : e->convs) {
    const int li = cv.level_in, lo = cv.level_out, cip = spconv_v6_cin_eff(cv.d.c_in);
    if (!cv.d.subm) nbrt = std::max(nbrt, (size_t)cv.kvol * caps[li]);
    wt = std::max(wt, (size_t)cv.kvol * cv.d.c_out * cip);
    if (enc_f16(e)) {   // the fp16 images are read in place: no widened or second image of dz
      pk = std::max(pk, spconv_v6_packed_bytes_f16(cv.d.c_out, cip, cv.kvol));
      wg = std::max(wg, spconv_wgrad_tc_f16_workspace_bytes(caps[lo], cv.d.c_in, cv.d.c_out, cv.kvol));
    } else {
      pk = std::max(pk, spconv_v6_packed_bytes(cv.d.c_out, cip, cv.kvol));
      wg = std::max(wg, spconv_wgrad_tc_split_workspace_bytes(caps[lo], cv.d.c_in, cv.d.c_out, cv.kvol));
      const int wide = spconv_wgrad_tc_image_channels(cv.d.c_in);
      if (wide != cip) fw = std::max(fw, (size_t)caps[li] * wide * 4);
      if (cv.d.c_out == 16) g16 = std::max(g16, (size_t)caps[lo] * 64);
    }
    part = std::max(part, (size_t)stat_chunks(caps[lo]) * 2 * cv.d.c_out);
    cmax = std::max(cmax, (size_t)cv.d.c_out);
  }
  b->nbr_t = a.take<int32_t>(nbrt);
  b->wt = a.take<float>(wt);
  b->packed = a.take<char>(pk);
  b->wg = a.take<char>(wg);
  b->fwide = a.take<uint8_t>(fw);
  b->g16 = a.take<uint8_t>(g16);
  b->din0 = a.take<float>((size_t)caps[0] * e->c0_eff);
  b->coef = a.take<float>(2 * cmax);
  b->partial = a.take<double>(part);
  return a.off;
}

}  // namespace bevb200

extern "C" {

size_t bevb200_encoder_train_state_bytes(const bevb200_encoder_t *e, int max_voxels, int batch_size,
                                         const int32_t *user_caps) {
  if (!e || enc_i8(e) || max_voxels <= 0 || batch_size <= 0) return 0;
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  ETrain t;
  return train_layout(e, caps, batch_size, nullptr, 0, &t);
}

int bevb200_encoder_train_saved(const bevb200_encoder_t *e, int max_voxels, int batch_size, const int32_t *user_caps,
                                int conv, size_t *pre_bn_offset, size_t *out_image_offset) {
  BEVB200_REQUIRE(e, "null plan");
  BEVB200_REQUIRE(!enc_i8(e), "an INT8 plan has no training path (eval forward only)");
  BEVB200_REQUIRE(max_voxels > 0 && batch_size > 0 && pre_bn_offset && out_image_offset, "bad argument");
  BEVB200_REQUIRE(conv >= 0 && conv < (int)e->convs.size(), "bad conv index");
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  // laid out from a stand-in base: every offset is pointer - base
  char *const base = (char *)(uintptr_t)4096;
  ETrain o;
  train_layout(e, caps, batch_size, base, 0, &o);
  *pre_bn_offset = (size_t)((char *)o.z[conv] - base);
  *out_image_offset = (size_t)((char *)o.y[conv] - base);
  return BEVB200_OK;
}

}  // extern "C"

static int enc_forward_train(bevb200_encoder_t *e, bool f16, const float *const *weights, const bevb200_encoder_bn_t *bn,
                             const void *voxel_features, const int32_t *coors, int max_voxels,
                             const int32_t *n_voxels_dev, int batch_size, const int32_t *user_caps, void *dense_out,
                             long long out_batch_stride, int32_t *status_dev, void *state, size_t state_bytes,
                             void *stream, void *rulebook_stream) {
  // the precision first: a call of the wrong family is refused before any other argument is looked at
  BEVB200_REQUIRE(e, "null plan");
  BEVB200_REQUIRE(!enc_i8(e), "an INT8 plan has no training path (eval forward only)");
  BEVB200_REQUIRE(enc_f16(e) == f16, f16 ? "the _f16 calls need a plan set to BEVB200_PREC_FP16"
                                         : "an fp16 plan runs the _f16 calls");
  BEVB200_REQUIRE(e && weights && bn && dense_out && status_dev && max_voxels > 0 && batch_size > 0, "bad argument");
  BEVB200_REQUIRE(voxel_features && coors, "null input");
  const size_t nc = e->convs.size();
  for (size_t i = 0; i < nc; ++i)
    BEVB200_REQUIRE(weights[i] && bn[i].weight && bn[i].bias && bn[i].running_mean && bn[i].running_var,
                    "null conv weight / BN tensor");
  cudaStream_t st = (cudaStream_t)stream, ss = rulebook_stream ? (cudaStream_t)rulebook_stream : st;
  const bool forked = ss != st;
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  ETrain t;
  const size_t need = train_layout(e, caps, batch_size, state, state_bytes, &t);
  if (state == nullptr || state_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "encoder_forward_train: state too small (%zu < %zu)", state_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  const size_t nl = e->levels.size(), nr = e->rulebooks.size();
  const EWs &w = t.w;
  int rc = enc_rulebooks(e, caps, max_voxels, batch_size, coors, n_voxels_dev, status_dev, w, st, ss);
  if (rc) return rc;
  // the live weights, packed on every call (a graph replay after an in-place optimizer step sees the new values)
  for (size_t i = 0; i < nc; ++i) {
    rc = enc_pack(e, e->convs[i], weights[i], t.params, st);
    if (rc) return rc;
  }
  rc = f16 ? spconv_v6_f16_rows((const __half *)voxel_features, caps[0], n_voxels_dev, e->in_channels, e->c0_eff,
                                t.in_split, st)
           : spconv_v6_split_rows((const float *)voxel_features, caps[0], n_voxels_dev, e->in_channels, e->c0_eff,
                                  t.in_split, st);
  if (rc) return rc;
  std::vector<char> rb_waited(nr, 0);
  const uint8_t *cur = t.in_split;
  for (size_t i = 0; i < nc; ++i) {
    const EConv &cv = e->convs[i];
    if (forked && !rb_waited[cv.rulebook]) {
      BEVB200_CUDA(cudaStreamWaitEvent(st, e->events[1 + cv.rulebook], 0));
      rb_waited[cv.rulebook] = 1;
    }
    const int lo = cv.level_out, c = cv.d.c_out;
    const bool last = i + 1 == nc;
    const uint8_t *res = cv.d.residual_from >= 0 ? t.y[cv.d.residual_from] : nullptr;
    const int grid = grid_for((long long)caps[lo] * (c / 8), 256);
    if (f16) {   // z16 = fp16(acc)
      rc = spconv_v6_forward_f16(cur, t.params + cv.packed_off, w.nbr[cv.rulebook], (long long)caps[lo],
                                 caps[cv.level_in], caps[lo], w.counts[lo], cv.c_in_eff, c, cv.kvol, nullptr, nullptr,
                                 nullptr, nullptr, 0, nullptr, t.z[i], st);
      if (rc) return rc;
      BEVB200_LAUNCH(bn_stats_partial_kernel<__half>, stat_chunks(caps[lo]), kStatThreads, 0, st,
                     (const __half *)t.z[i], w.counts[lo], caps[lo], c, t.partial);
    } else {
      rc = spconv_v6_forward(cur, t.params + cv.packed_off, w.nbr[cv.rulebook], (long long)caps[lo], caps[cv.level_in],
                             caps[lo], w.counts[lo], cv.c_in_eff, c, cv.kvol, nullptr, nullptr, nullptr, nullptr, 0,
                             (float *)t.z[i], nullptr, st);
      if (rc) return rc;
      BEVB200_LAUNCH(bn_stats_partial_kernel<float>, stat_chunks(caps[lo]), kStatThreads, 0, st, (const float *)t.z[i],
                     w.counts[lo], caps[lo], c, t.partial);
    }
    BEVB200_LAUNCH(bn_stats_reduce_kernel, 1, kStatThreads, 0, st, t.partial, w.counts[lo], caps[lo], c, bn[i],
                   t.stat[i], status_dev);
    if (f16)
      BEVB200_LAUNCH(bn_apply_kernel<true>, grid, 256, 0, st, (const __half *)t.z[i], t.stat[i], res, w.counts[lo],
                     caps[lo], c, cv.d.relu, t.y[i], (float *)nullptr);
    else
      BEVB200_LAUNCH(bn_apply_kernel<false>, grid, 256, 0, st, (const float *)t.z[i], t.stat[i], res, w.counts[lo],
                     caps[lo], c, cv.d.relu, t.y[i], last ? t.y_last : nullptr);
    cur = t.y[i];
  }
  const size_t ll = nl - 1;
  const int32_t *lidx = w.indices[ll] ? w.indices[ll] : coors;
  rc = f16 ? sparse_to_dense((const __half *)cur, lidx, caps[ll], w.counts[ll], e->convs.back().d.c_out, batch_size,
                             e->levels[ll].shape, 1, out_batch_stride, (__half *)dense_out, st)
           : sparse_to_dense(t.y_last, lidx, caps[ll], w.counts[ll], e->convs.back().d.c_out, batch_size,
                             e->levels[ll].shape, 1, out_batch_stride, (float *)dense_out, st);
  if (rc) return rc;
  if (forked) BEVB200_CUDA(cudaStreamWaitEvent(st, e->events[1 + nr], 0));
  return BEVB200_OK;
}

extern "C" {

int bevb200_encoder_forward_train(bevb200_encoder_t *e, const float *const *weights, const bevb200_encoder_bn_t *bn,
                                  const float *voxel_features, const int32_t *coors, int max_voxels,
                                  const int32_t *n_voxels_dev, int batch_size, const int32_t *user_caps,
                                  float *dense_out, long long out_batch_stride, int32_t *status_dev, void *state,
                                  size_t state_bytes, void *stream, void *rulebook_stream) {
  return enc_forward_train(e, false, weights, bn, voxel_features, coors, max_voxels, n_voxels_dev, batch_size,
                           user_caps, dense_out, out_batch_stride, status_dev, state, state_bytes, stream,
                           rulebook_stream);
}

int bevb200_encoder_forward_train_f16(bevb200_encoder_t *e, const float *const *weights,
                                      const bevb200_encoder_bn_t *bn, const void *voxel_features,
                                      const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev,
                                      int batch_size, const int32_t *user_caps, void *dense_out,
                                      long long out_batch_stride, int32_t *status_dev, void *state,
                                      size_t state_bytes, void *stream, void *rulebook_stream) {
  return enc_forward_train(e, true, weights, bn, voxel_features, coors, max_voxels, n_voxels_dev, batch_size,
                           user_caps, dense_out, out_batch_stride, status_dev, state, state_bytes, stream,
                           rulebook_stream);
}

size_t bevb200_encoder_backward_workspace_bytes(const bevb200_encoder_t *e, int max_voxels, int batch_size,
                                                const int32_t *user_caps) {
  if (!e || enc_i8(e) || max_voxels <= 0 || batch_size <= 0) return 0;
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  EBwd b;
  return bwd_layout(e, caps, nullptr, 0, &b);
}

}  // extern "C"

static int enc_backward(const bevb200_encoder_t *e, bool f16, const float *const *weights, const void *state,
                        size_t state_bytes, int max_voxels, int batch_size, const int32_t *user_caps,
                        const void *grad_dense, long long out_batch_stride, void *grad_voxel_features,
                        float *const *grad_weights, float *const *grad_bn_weight, float *const *grad_bn_bias,
                        void *workspace, size_t workspace_bytes, void *stream) {
  // the precision first: a call of the wrong family is refused before any other argument is looked at
  BEVB200_REQUIRE(e, "null plan");
  BEVB200_REQUIRE(!enc_i8(e), "an INT8 plan has no training path (eval forward only)");
  BEVB200_REQUIRE(enc_f16(e) == f16, f16 ? "the _f16 calls need a plan set to BEVB200_PREC_FP16"
                                         : "an fp16 plan runs the _f16 calls");
  BEVB200_REQUIRE(e && weights && state && grad_dense && grad_weights && grad_bn_weight && grad_bn_bias &&
                      max_voxels > 0 && batch_size > 0, "bad argument");
  const size_t nc = e->convs.size(), nl = e->levels.size();
  for (size_t i = 0; i < nc; ++i)
    BEVB200_REQUIRE(weights[i] && grad_weights[i] && grad_bn_weight[i] && grad_bn_bias[i], "null conv / BN tensor");
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<int> caps;
  level_caps(e, max_voxels, batch_size, user_caps, &caps);
  ETrain t;
  const size_t need_state = train_layout(e, caps, batch_size, (void *)state, state_bytes, &t);
  BEVB200_REQUIRE(state_bytes >= need_state, "state smaller than train_state_bytes");
  EBwd b;
  const size_t need = bwd_layout(e, caps, workspace, workspace_bytes, &b);
  if (workspace == nullptr || workspace_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "encoder_backward: workspace too small (%zu < %zu)", workspace_bytes, need);
    return BEVB200_EWORKSPACE;
  }
  const EWs &w = t.w;
  if (out_batch_stride == 0) {
    const int *s = e->levels.back().shape;
    out_batch_stride = (long long)e->convs.back().d.c_out * s[0] * s[1] * s[2];
  }
  // the last level's rows from the dense gradient
  const size_t ll = nl - 1;
  BEVB200_REQUIRE(ll > 0, "a plan without a strided conv has no training path");
  {
    const int *s = e->levels[ll].shape;
    const int c = e->convs.back().d.c_out;
    if (f16)
      BEVB200_LAUNCH(dense_gather_kernel<__half>, grid_for((long long)caps[ll] * c, 256), 256, 0, st,
                     (const __half *)grad_dense, w.indices[ll], w.counts[ll], caps[ll], c, batch_size, s[0], s[1], s[2],
                     out_batch_stride, b.d[0][ll]);
    else
      BEVB200_LAUNCH(dense_gather_kernel<float>, grid_for((long long)caps[ll] * c, 256), 256, 0, st,
                     (const float *)grad_dense, w.indices[ll], w.counts[ll], caps[ll], c, batch_size, s[0], s[1], s[2],
                     out_batch_stride, b.d[0][ll]);
  }
  std::vector<int> cur(nl, 0), held(nl, -1);
  const float *pending = nullptr;   // a block's identity gradient, added to the input gradient of conv pending_for
  int pending_for = -1;
  int rc;
  for (int i = (int)nc - 1; i >= 0; --i) {
    const EConv &cv = e->convs[i];
    const int lo = cv.level_out, li = cv.level_in, c = cv.d.c_out;
    const bool last = i + 1 == (int)nc;
    float *g = b.d[cur[lo]][lo];
    // ReLU mask, BN backward
    if (f16)
      BEVB200_LAUNCH(bn_bwd_partial_kernel<true>, stat_chunks(caps[lo]), kStatThreads, 0, st, g, t.y[i],
                     (const float *)nullptr, cv.d.relu, (const __half *)t.z[i], t.stat[i], w.counts[lo], caps[lo], c,
                     b.partial);
    else
      BEVB200_LAUNCH(bn_bwd_partial_kernel<false>, stat_chunks(caps[lo]), kStatThreads, 0, st, g, t.y[i],
                     last ? t.y_last : nullptr, cv.d.relu, (const float *)t.z[i], t.stat[i], w.counts[lo], caps[lo], c,
                     b.partial);
    BEVB200_LAUNCH(bn_bwd_reduce_kernel, 1, kStatThreads, 0, st, b.partial, w.counts[lo], caps[lo], c,
                   grad_bn_weight[i], grad_bn_bias[i], b.coef);
    if (f16)
      BEVB200_LAUNCH(bn_bwd_apply_kernel<true>, grid_for((long long)caps[lo] * c, 256), 256, 0, st, g,
                     (const __half *)t.z[i], t.stat[i], b.coef, w.counts[lo], caps[lo], c, (__half *)b.dz[lo]);
    else
      BEVB200_LAUNCH(bn_bwd_apply_kernel<false>, grid_for((long long)caps[lo] * c, 256), 256, 0, st, g,
                     (const float *)t.z[i], t.stat[i], b.coef, w.counts[lo], caps[lo], c, (float *)b.dz[lo]);
    if (cv.d.residual_from >= 0) {   // g (after the mask) is also the gradient of the identity
      BEVB200_REQUIRE(pending_for < 0, "two pending residual gradients");
      held[lo] = cur[lo];
      pending = g;
      pending_for = cv.d.residual_from + 1;
    }
    // filter gradient on the saved input image
    const int cip = spconv_v6_cin_eff(cv.d.c_in), wide = spconv_wgrad_tc_image_channels(cv.d.c_in);
    const uint8_t *fimg = i == 0 ? t.in_split : t.y[i - 1];
    if (f16) {
      rc = spconv_wgrad_tc_f16(fimg, cip, b.dz[lo], w.nbr[cv.rulebook], caps[li], caps[lo], w.counts[lo], cv.d.c_in, c,
                               cv.kvol, grad_weights[i], b.wg, st);
    } else {
      if (wide != cip) {
        BEVB200_LAUNCH(enc_widen_image_kernel, grid_for((long long)caps[li] * (wide / 4), 256), 256, 0, st, fimg, cip,
                       wide, w.counts[li], caps[li], b.fwide);
        fimg = b.fwide;
      }
      rc = spconv_wgrad_tc_split(fimg, (const float *)b.dz[lo], w.nbr[cv.rulebook], caps[li], caps[lo], w.counts[lo],
                                 cv.d.c_in, c, cv.kvol, grad_weights[i], b.wg, st);
    }
    if (rc) return rc;
    // input gradient
    if (i == 0 && grad_voxel_features == nullptr) break;
    BEVB200_LAUNCH(enc_weight_t_kernel, grid_for((long long)cv.kvol * c * cip, 256), 256, 0, st, weights[i], cv.kvol,
                   cv.d.c_in, c, cip, cv.d.subm, b.wt);
    rc = f16 ? spconv_v6_pack_weights_f16(b.wt, c, cip, cv.kvol, b.packed, st)
             : spconv_v6_pack_weights(b.wt, c, cip, cv.kvol, b.packed, st);
    if (rc) return rc;
    const void *gimg = b.wg;   // c_out 32 / 64 / 128: the filter gradient's image of dz is the forward's row image
    if (f16) {
      gimg = b.dz[lo];         // the one fp16 image of dz
    } else if (c == 16) {
      rc = spconv_v6_split_rows((const float *)b.dz[lo], caps[lo], w.counts[lo], c, c, b.g16, st);
      if (rc) return rc;
      gimg = b.g16;
    }
    const int32_t *table = w.nbr[cv.rulebook];   // SubM: the forward table with mirrored offsets (in the weights)
    if (!cv.d.subm) {
      BEVB200_LAUNCH(enc_nbr_t_fill_kernel, grid_for((long long)cv.kvol * caps[li], 256), 256, 0, st, w.counts[li],
                     caps[li], cv.kvol, b.nbr_t);
      BEVB200_LAUNCH(enc_nbr_t_scatter_kernel, grid_for((long long)cv.kvol * caps[lo], 256), 256, 0, st,
                     w.nbr[cv.rulebook], w.counts[lo], caps[lo], w.counts[li], caps[li], cv.kvol, b.nbr_t);
      table = b.nbr_t;
    }
    const float *res = pending_for == i ? pending : nullptr;
    float *out;
    int oi = 0;
    if (i == 0) {
      out = b.din0;
    } else {
      oi = (li == lo && held[lo] == cur[lo]) ? cur[lo] ^ 1 : (li == lo ? cur[lo] : 0);
      out = b.d[oi][li];
    }
    rc = (f16 ? spconv_v6_forward_f16 : spconv_v6_forward)(gimg, b.packed, table, (long long)caps[li], caps[lo],
                                                           caps[li], w.counts[li], c, cip, cv.kvol, nullptr, nullptr,
                                                           res, nullptr, 0, out, nullptr, st);
    if (rc) return rc;
    if (res) {
      pending = nullptr;
      pending_for = -1;
      held[lo] = -1;
    }
    if (i == 0) {
      if (f16)
        BEVB200_LAUNCH(enc_narrow_grad_kernel<__half>, grid_for((long long)max_voxels * e->in_channels, 256), 256, 0,
                       st, b.din0, e->c0_eff, w.counts[0], caps[0], max_voxels, e->in_channels,
                       (__half *)grad_voxel_features);
      else
        BEVB200_LAUNCH(enc_narrow_grad_kernel<float>, grid_for((long long)max_voxels * e->in_channels, 256), 256, 0,
                       st, b.din0, e->c0_eff, w.counts[0], caps[0], max_voxels, e->in_channels,
                       (float *)grad_voxel_features);
    } else {
      cur[li] = oi;
    }
  }
  return BEVB200_OK;
}

extern "C" {

int bevb200_encoder_backward(const bevb200_encoder_t *e, const float *const *weights, const void *state,
                             size_t state_bytes, int max_voxels, int batch_size, const int32_t *user_caps,
                             const float *grad_dense, long long out_batch_stride, float *grad_voxel_features,
                             float *const *grad_weights, float *const *grad_bn_weight, float *const *grad_bn_bias,
                             void *workspace, size_t workspace_bytes, void *stream) {
  return enc_backward(e, false, weights, state, state_bytes, max_voxels, batch_size, user_caps, grad_dense,
                      out_batch_stride, grad_voxel_features, grad_weights, grad_bn_weight, grad_bn_bias, workspace,
                      workspace_bytes, stream);
}

int bevb200_encoder_backward_f16(const bevb200_encoder_t *e, const float *const *weights, const void *state,
                                 size_t state_bytes, int max_voxels, int batch_size, const int32_t *user_caps,
                                 const void *grad_dense, long long out_batch_stride, void *grad_voxel_features,
                                 float *const *grad_weights, float *const *grad_bn_weight,
                                 float *const *grad_bn_bias, void *workspace, size_t workspace_bytes, void *stream) {
  return enc_backward(e, true, weights, state, state_bytes, max_voxels, batch_size, user_caps, grad_dense,
                      out_batch_stride, grad_voxel_features, grad_weights, grad_bn_weight, grad_bn_bias, workspace,
                      workspace_bytes, stream);
}

}  // extern "C"
