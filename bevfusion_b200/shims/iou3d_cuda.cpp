// Drop-in for the reference's pybind module `iou3d_cuda` (mmdet3d/ops/iou3d/src/iou3d.cpp:48-216): same
// names, argument order and return values, each a thin shim over the C ABI of libbevfusion_b200.  As in the
// reference, `keep` of nms_gpu / nms_normal_gpu is a CPU int64 tensor and the return value is the kept
// count.  There is no CPU path: CPU boxes raise.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "bevfusion_b200.h"

namespace {
void check_input(const at::Tensor &t, const char *name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor: bevfusion_b200 has no CPU path");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
  TORCH_CHECK(t.scalar_type() == at::kFloat, name, " must be float32");
}
cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

int dense(const at::Tensor &a, const at::Tensor &b, at::Tensor &out, bool iou) {
  check_input(a, "boxes_a"); check_input(b, "boxes_b"); check_input(out, "ans");
  TORCH_CHECK(out.numel() == a.size(0) * b.size(0), "ans must hold boxes_a.size(0) * boxes_b.size(0) values");
  c10::cuda::CUDAGuard guard(a.device());
  const int rc = (iou ? bevb200_boxes_iou_bev : bevb200_boxes_overlap_bev)(
      a.data_ptr<float>(), a.size(0), b.data_ptr<float>(), b.size(0), out.data_ptr<float>(), cur_stream());
  TORCH_CHECK(rc == 0, bevb200_last_error());
  return 1;
}

int nms(const at::Tensor &boxes, at::Tensor &keep, float thresh, int mode) {
  check_input(boxes, "boxes");
  TORCH_CHECK(keep.is_contiguous() && keep.scalar_type() == at::kLong, "keep must be a contiguous int64 tensor");
  const int n = boxes.size(0);
  TORCH_CHECK(keep.numel() >= n, "keep must hold boxes.size(0) values");
  c10::cuda::CUDAGuard guard(boxes.device());
  auto opts = boxes.options();
  auto keep_dev = at::empty({1, n}, opts.dtype(at::kLong));
  auto count = at::empty({1}, opts.dtype(at::kInt));
  const size_t ws_bytes = bevb200_nms_workspace_bytes(1, n);
  auto ws = at::empty({(int64_t)ws_bytes + 1}, opts.dtype(at::kByte));
  const int rc = bevb200_nms(boxes.data_ptr<float>(), nullptr, 1, n, mode, (double)thresh, n, nullptr,
                             keep_dev.data_ptr<int64_t>(), count.data_ptr<int32_t>(), ws.data_ptr(), ws_bytes,
                             cur_stream());
  TORCH_CHECK(rc == 0, bevb200_last_error());
  const int num = count.item<int>();
  if (num > 0) keep.narrow(0, 0, num).copy_(keep_dev[0].narrow(0, 0, num));
  return num;
}

// Internal linkage: the reference's own module (same function names) may be loaded in the same process.
int boxes_overlap_bev_gpu(at::Tensor boxes_a, at::Tensor boxes_b, at::Tensor ans_overlap) {
  return dense(boxes_a, boxes_b, ans_overlap, false);
}

int boxes_iou_bev_gpu(at::Tensor boxes_a, at::Tensor boxes_b, at::Tensor ans_iou) {
  return dense(boxes_a, boxes_b, ans_iou, true);
}

int nms_gpu(at::Tensor boxes, at::Tensor keep, float nms_overlap_thresh, int device_id) {
  TORCH_CHECK(boxes.is_cuda() && boxes.get_device() == device_id, "boxes must be a CUDA tensor on device_id");
  return nms(boxes, keep, nms_overlap_thresh, BEVB200_NMS_ROTATE);
}

int nms_normal_gpu(at::Tensor boxes, at::Tensor keep, float nms_overlap_thresh, int device_id) {
  TORCH_CHECK(boxes.is_cuda() && boxes.get_device() == device_id, "boxes must be a CUDA tensor on device_id");
  return nms(boxes, keep, nms_overlap_thresh, BEVB200_NMS_NORMAL);
}
}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("boxes_overlap_bev_gpu", &boxes_overlap_bev_gpu, "oriented boxes overlap");
  m.def("boxes_iou_bev_gpu", &boxes_iou_bev_gpu, "oriented boxes iou");
  m.def("nms_gpu", &nms_gpu, "oriented nms gpu");
  m.def("nms_normal_gpu", &nms_normal_gpu, "nms gpu");
}
