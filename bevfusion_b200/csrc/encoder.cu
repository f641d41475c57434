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
  std::vector<EConv> convs;
  std::vector<ELevel> levels;
  std::vector<ERulebook> rulebooks;
  size_t param_bytes;
  std::vector<cudaEvent_t> events;   // [0] fork, [1..] one per rulebook, last: join
  int event_device;
};

namespace bevb200 {

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
  char *zero_begin, *zero_end;
  size_t bytes;
};

static size_t enc_layout(const bevb200_encoder *e, const std::vector<int> &caps, int batch, void *ws, size_t ws_bytes,
                         EWs *w) {
  Arena a(ws, ws_bytes);
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
    w->split[s].resize(nl);
    w->f32[s].resize(nl);
    for (size_t l = 0; l < nl; ++l) {
      const size_t row = (size_t)e->levels[l].c_max * 4;
      w->split[s][l] = a.take<uint8_t>((size_t)caps[l] * row);
      w->f32[s][l] = a.take<float>((size_t)caps[l] * e->levels[l].c_max);
    }
  }
  w->bytes = a.off;
  return a.off;
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
  e->event_device = -1;
  ELevel l0;
  for (int d = 0; d < 3; ++d) l0.shape[d] = sparse_shape_host[d];
  l0.c_max = e->c0_eff;
  e->levels.push_back(l0);
  int level = 0, c_prev = in_channels;
  size_t poff = 0;
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
    cv.packed_off = poff; poff += align_up(spconv_v6_packed_bytes(cv.d.c_in, cv.d.c_out, cv.kvol));
    cv.scale_off = poff; poff += align_up((size_t)cv.d.c_out * 4);
    cv.shift_off = poff; poff += align_up((size_t)cv.d.c_out * 4);
    cv.has_scale = cv.has_shift = false;
    e->convs.push_back(cv);
    c_prev = cv.d.c_out;
  }
  // A residual is read from the source conv's SPLIT image -- hi + lo is the value to 2^-17 -- so only the last conv,
  // whose rows dense() scatters, writes fp32 rows; BEVB200_ENCODER_F32_RESIDUAL=1 restores the fp32 residual copies.
  static const bool f32_residual = [] { const char *v = getenv("BEVB200_ENCODER_F32_RESIDUAL"); return v && atoi(v) != 0; }();
  for (EConv &cv : e->convs)
    if (f32_residual && cv.d.residual_from >= 0) e->convs[cv.d.residual_from].want_fp32 = true;
  e->param_bytes = poff;
  *out = e;
  return BEVB200_OK;
}

void bevb200_encoder_destroy(bevb200_encoder_t *e) {
  if (!e) return;
  for (cudaEvent_t ev : e->events) cudaEventDestroy(ev);
  delete e;
}

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
  BEVB200_REQUIRE(weight && params && params_bytes >= e->param_bytes, "null argument / parameter buffer too small");
  EConv &cv = e->convs[conv];
  cudaStream_t st = (cudaStream_t)stream;
  char *base = (char *)params;
  int rc = spconv_v6_pack_weights(weight, cv.d.c_in, cv.d.c_out, cv.kvol, base + cv.packed_off, st);
  if (rc) return rc;
  cv.has_scale = scale != nullptr;
  cv.has_shift = shift != nullptr;
  if (scale)
    BEVB200_CUDA(cudaMemcpyAsync(base + cv.scale_off, scale, (size_t)cv.d.c_out * 4, cudaMemcpyDeviceToDevice, st));
  if (shift)
    BEVB200_CUDA(cudaMemcpyAsync(base + cv.shift_off, shift, (size_t)cv.d.c_out * 4, cudaMemcpyDeviceToDevice, st));
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

int bevb200_encoder_forward(bevb200_encoder_t *e, const void *params, const float *voxel_features,
                            const int32_t *coors, int max_voxels, const int32_t *n_voxels_dev, int batch_size,
                            const int32_t *user_caps, float *dense_out, long long out_batch_stride,
                            int32_t *status_dev, void *workspace, size_t workspace_bytes, void *stream,
                            void *rulebook_stream) {
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
  const char *pbase = (const char *)params;
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

  // ------------------------------ rulebooks (stream ss) ------------------------------------
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

  // ------------------------------ features (stream st) -------------------------------------
  int rc = spconv_v6_split_rows(voxel_features, caps[0], n_voxels_dev, e->in_channels, e->c0_eff, w.split[0][0], st);
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
    if (!last) {
      osplit = w.split[split_turn[lo]][lo];
      split_turn[lo] ^= 1;
    }
    float *of32 = nullptr;
    if (cv.want_fp32) {
      of32 = w.f32[f32_turn[lo]][lo];
      f32_turn[lo] ^= 1;
      f32_of[i] = of32;
    }
    // residual: the source conv's fp32 rows if it wrote them, else its split image (which may be the buffer this conv
    // writes: the two split buffers of a level alternate and a block's input is two convs back -- safe, see spconv_v6.cu)
    const float *res = cv.d.residual_from >= 0 ? f32_of[cv.d.residual_from] : nullptr;
    const uint8_t *res_split = (cv.d.residual_from >= 0 && res == nullptr) ? split_of[cv.d.residual_from] : nullptr;
    BEVB200_REQUIRE(cv.d.residual_from < 0 || res || res_split, "residual source has no rows");
    rc = spconv_v6_forward(cur_split, pbase + cv.packed_off, w.nbr[cv.rulebook], (long long)caps[lo], caps[cv.level_in],
                           caps[lo], w.counts[lo], cv.c_in_eff, cv.d.c_out, cv.kvol,
                           cv.has_scale ? (const float *)(pbase + cv.scale_off) : nullptr,
                           cv.has_shift ? (const float *)(pbase + cv.shift_off) : nullptr, res, res_split, cv.d.relu,
                           of32, osplit, st);
    if (rc) return rc;
    split_of[i] = osplit;
    cur_split = osplit;
    last_f32 = of32;
  }
  // dense(): [B, C*Z, X, Y]
  const size_t ll = nl - 1;
  rc = sparse_to_dense(last_f32, w.indices[ll] ? w.indices[ll] : idx0, caps[ll], w.counts[ll], e->convs.back().d.c_out,
                       batch_size, e->levels[ll].shape, 1, out_batch_stride, dense_out, st);
  if (rc) return rc;
  if (forked) BEVB200_CUDA(cudaStreamWaitEvent(st, e->events[1 + nr], 0));   // join (also what a graph capture needs)
  return BEVB200_OK;
}

}  // extern "C"
