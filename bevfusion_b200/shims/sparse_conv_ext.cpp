// Drop-in for the reference's pybind module `sparse_conv_ext` (mmdet3d/ops/spconv/src/all.cc:22-50): the
// names a 3-D model reaches -- get_indice_pairs_3d (spconv_ops.h:27-141), indice_conv_{fp32,half} (:260-361),
// indice_conv_backward_{fp32,half} (:363-456), fused_indice_conv_{fp32,half} (fused_spconv_ops.h:28-131) --
// with the reference's argument order and return layouts, each a thin shim over the C ABI of
// libbevfusion_b200.  2-D / 4-D / grid rulebooks and sparse max-pool are not provided (no shipped
// BEVFusion config reaches them).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <vector>

#include "bevfusion_b200.h"

namespace {
cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
void check_cuda(const torch::Tensor &t, const char *name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor: bevfusion_b200 has no CPU path");
}
std::vector<int32_t> i32(const std::vector<int64_t> &v) { return std::vector<int32_t>(v.begin(), v.end()); }

torch::Tensor nbr_of(const torch::Tensor &indicePairs, const torch::Tensor &indiceNum, int64_t numActOut, int64_t inverse) {
  const int K = indicePairs.size(0);
  auto pairs = indicePairs.contiguous();
  auto num = indiceNum.contiguous();
  auto nbr = torch::empty({K, numActOut}, pairs.options());
  TORCH_CHECK(0 == bevb200_pairs_to_nbr(pairs.data_ptr<int>(), num.data_ptr<int>(), K, (int)pairs.size(2), (int)numActOut,
                                        (int)inverse, nbr.data_ptr<int>(), cur_stream()),
              bevb200_last_error());
  return nbr;
}
}  // namespace

std::vector<torch::Tensor> get_indice_pairs_3d(torch::Tensor indices, int64_t batchSize, std::vector<int64_t> outSpatialShape,
                                               std::vector<int64_t> spatialShape, std::vector<int64_t> kernelSize,
                                               std::vector<int64_t> stride, std::vector<int64_t> padding,
                                               std::vector<int64_t> dilation, std::vector<int64_t> outPadding,
                                               int64_t _subM, int64_t _transpose) {
  check_cuda(indices, "indices");
  TORCH_CHECK(!_transpose, "transposed sparse conv is outside the hot path");
  TORCH_CHECK(indices.dim() == 2 && indices.size(1) == 4 && kernelSize.size() == 3, "3-D sparse conv only");
  (void)outPadding;
  c10::cuda::CUDAGuard guard(indices.device());
  indices = indices.contiguous();
  auto s = i32(spatialShape), o = i32(outSpatialShape), k = i32(kernelSize), st = i32(stride), p = i32(padding), d = i32(dilation);
  const int n = indices.size(0), K = k[0] * k[1] * k[2];
  const int subM = _subM != 0;
  auto ws = torch::empty({(int64_t)bevb200_rulebook_workspace_bytes(n, (int)batchSize, o.data()) + 256},
                         indices.options().dtype(torch::kUInt8));
  auto nOut = torch::zeros({1}, indices.options());
  TORCH_CHECK(0 == bevb200_rulebook_prepare(indices.data_ptr<int>(), n, (int)batchSize, s.data(), o.data(), k.data(), st.data(),
                                            p.data(), d.data(), subM, nOut.data_ptr<int>(), ws.data_ptr(), (size_t)ws.numel(),
                                            cur_stream()),
              bevb200_last_error());
  const int m = subM ? n : nOut.item<int>();     // the reference syncs here too (spconv_ops.h:113-118)
  auto outInds = subM ? indices : torch::empty({m, 4}, indices.options());
  auto nbr = torch::empty({K, m}, indices.options());
  TORCH_CHECK(0 == bevb200_rulebook_fill(indices.data_ptr<int>(), n, (int)batchSize, s.data(), o.data(), k.data(), st.data(),
                                         p.data(), d.data(), subM, m, outInds.data_ptr<int>(), nbr.data_ptr<int>(),
                                         ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
              bevb200_last_error());
  auto pairs = torch::empty({K, 2, n}, indices.options());
  auto num = torch::empty({K}, indices.options());
  TORCH_CHECK(0 == bevb200_rulebook_to_pairs(nbr.data_ptr<int>(), K, m, n, pairs.data_ptr<int>(), num.data_ptr<int>(), cur_stream()),
              bevb200_last_error());
  return {outInds, pairs, num};
}

// half tensors are widened, computed with fp32 accumulation on the tensor cores and narrowed once; the
// output is half when the features or the filters are (the rule of the python module's indice_conv)
static torch::Tensor conv_impl(torch::Tensor features, torch::Tensor filters, const torch::Tensor *bias,
                               torch::Tensor indicePairs, torch::Tensor indiceNum, int64_t numActOut, int64_t inverse) {
  check_cuda(features, "features"); check_cuda(filters, "filters"); check_cuda(indicePairs, "indicePairs");
  c10::cuda::CUDAGuard guard(features.device());
  const bool half = features.scalar_type() == torch::kHalf || filters.scalar_type() == torch::kHalf;
  const auto in_dtype = half ? torch::kHalf : features.scalar_type();
  auto f = features.to(torch::kFloat32).contiguous();
  auto w = filters.to(torch::kFloat32).contiguous();
  const int K = indicePairs.size(0), cin = f.size(1), cout = w.size(w.dim() - 1);
  auto nbr = nbr_of(indicePairs, indiceNum, numActOut, inverse);
  auto out = torch::empty({numActOut, cout}, f.options());
  torch::Tensor b;
  if (bias) b = bias->to(torch::kFloat32).contiguous();
  TORCH_CHECK(0 == bevb200_spconv_forward(f.data_ptr<float>(), w.data_ptr<float>(), nbr.data_ptr<int>(), (int)f.size(0),
                                          (int)numActOut, cin, cout, K, nullptr, bias ? b.data_ptr<float>() : nullptr, nullptr,
                                          0, BEVB200_PREC_BF16X3, out.data_ptr<float>(), cur_stream()),
              bevb200_last_error());
  return out.to(in_dtype);
}

torch::Tensor indice_conv(torch::Tensor features, torch::Tensor filters, torch::Tensor indicePairs, torch::Tensor indiceNum,
                          int64_t numActOut, int64_t _inverse, int64_t _subM) {
  (void)_subM;   // the centre offset of a SubM conv is just another column of the neighbour table
  return conv_impl(features, filters, nullptr, indicePairs, indiceNum, numActOut, _inverse);
}

torch::Tensor fused_indice_conv(torch::Tensor features, torch::Tensor filters, torch::Tensor bias, torch::Tensor indicePairs,
                                torch::Tensor indiceNum, int64_t numActOut, int64_t _inverse, int64_t _subM) {
  (void)_subM;
  return conv_impl(features, filters, &bias, indicePairs, indiceNum, numActOut, _inverse);
}

std::vector<torch::Tensor> indice_conv_backward(torch::Tensor features, torch::Tensor filters, torch::Tensor outGrad,
                                                torch::Tensor indicePairs, torch::Tensor indiceNum, int64_t _inverse,
                                                int64_t _subM) {
  (void)_subM;
  check_cuda(features, "features"); check_cuda(filters, "filters"); check_cuda(outGrad, "outGrad");
  c10::cuda::CUDAGuard guard(features.device());
  // each gradient in the dtype of the tensor it belongs to
  const auto f_dtype = features.scalar_type(), w_dtype = filters.scalar_type();
  auto f = features.to(torch::kFloat32).contiguous();
  auto w = filters.to(torch::kFloat32).contiguous();
  auto g = outGrad.to(torch::kFloat32).contiguous();
  const int K = indicePairs.size(0), n_in = f.size(0), n_out = g.size(0), cin = f.size(1), cout = w.size(w.dim() - 1);
  auto nbr = nbr_of(indicePairs, indiceNum, n_out, _inverse);
  auto nbr_t = torch::empty({K, n_in}, nbr.options());
  TORCH_CHECK(0 == bevb200_rulebook_transpose(nbr.data_ptr<int>(), K, n_out, n_in, nbr_t.data_ptr<int>(), cur_stream()),
              bevb200_last_error());
  auto din = torch::empty({n_in, cin}, f.options());
  auto dw = torch::empty_like(w);
  auto ws = torch::empty({(int64_t)bevb200_spconv_backward_workspace_bytes(n_in, n_out, cin, cout, K) + 256}, f.options().dtype(torch::kUInt8));
  TORCH_CHECK(0 == bevb200_spconv_backward(f.data_ptr<float>(), w.data_ptr<float>(), g.data_ptr<float>(), nbr.data_ptr<int>(),
                                           nbr_t.data_ptr<int>(), n_in, n_out, cin, cout, K, BEVB200_PREC_BF16X3,
                                           din.data_ptr<float>(), dw.data_ptr<float>(), ws.data_ptr(), (size_t)ws.numel(),
                                           cur_stream()),
              bevb200_last_error());
  return {din.to(f_dtype), dw.to(w_dtype)};
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("get_indice_pairs_3d", &get_indice_pairs_3d, "get_indice_pairs_3d");
  m.def("indice_conv_fp32", &indice_conv, "indice_conv_fp32");
  m.def("indice_conv_half", &indice_conv, "indice_conv_half");
  m.def("indice_conv_backward_fp32", &indice_conv_backward, "indice_conv_backward_fp32");
  m.def("indice_conv_backward_half", &indice_conv_backward, "indice_conv_backward_half");
  m.def("fused_indice_conv_fp32", &fused_indice_conv, "fused_indice_conv_fp32");
  m.def("fused_indice_conv_half", &fused_indice_conv, "fused_indice_conv_half");
}
