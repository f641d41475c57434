"""transfusion_proposals -- the query initialisation of TransFusionHead.forward_single on the device
(csrc/transfusion_proposals.cu): sigmoid of the dense heatmap, the k x k peak mask, the top num_proposals of the
masked plane and the query_heatmap_score gather (transfusion.py:237-281 and :322-325), in one native call.

    transfusion_proposals(dense_heatmap, num_proposals, nms_kernel_size=3, dataset="nuScenes")
        -> (labels [B, K] int64, index [B, K] int64, query_heatmap_score [B, C, K] in the heatmap's dtype)

Two launches, no host synchronisation, no allocation inside the call beyond its outputs and workspace; CUDA-graph
capturable and the same bit for bit on every run.  labels is the reference's self.query_labels; the head keeps its
two gathers (query_feat from the flattened LiDAR features, query_pos from bev_pos) on `index` with their autograd.

Semantics: s = sigmoid(x) as torch computes it on CUDA, in x's dtype; local_max = the k x k window maximum (NaN
propagates) on cells at least k // 2 from every edge, 0 in the border band, and s itself for the dataset's exempt
classes (nuScenes 8, 9; Waymo 1, 2; none otherwise); m = s * (s == local_max).  The top K of the C * H * W values of
m per sample are taken in descending value, NaN first, ties by ascending flat index c * H * W + h * W + w: the
reference's argsort with stable=True (its own argsort is unstable, so its tie order is unspecified).  The heatmap is
detached in the reference; there is no autograd here.  GPU only: CPU tensors raise."""
import torch

from . import _C

__all__ = ["transfusion_proposals", "exempt_classes", "workspace_bytes", "MAX_CLASSES", "MAX_PROPOSALS",
           "MAX_KERNEL", "MAX_CELLS", "MAX_BATCH"]

MAX_BATCH = 65535          # BEVB200_PROPOSALS_MAX_BATCH
MAX_CLASSES = 64           # BEVB200_PROPOSALS_MAX_CLASSES
MAX_CELLS = 1 << 24        # BEVB200_PROPOSALS_MAX_CELLS, C * H * W per sample
MAX_PROPOSALS = 4096       # BEVB200_PROPOSALS_MAX_K
MAX_KERNEL = 15            # BEVB200_PROPOSALS_MAX_KERNEL

_DTYPES = {torch.float32: 0, torch.float16: 1}   # BEVB200_PROPOSALS_F32 / _F16


def exempt_classes(dataset):
    """The classes whose peak test is against themselves: test_cfg['dataset'] "nuScenes" -> (8, 9) (pedestrian,
    traffic cone), "Waymo" -> (1, 2) (pedestrian, cyclist), anything else -> ()."""
    if dataset == "nuScenes":
        return (8, 9)
    if dataset == "Waymo":
        return (1, 2)
    return ()


def workspace_bytes(B, C, H, W):
    """Device workspace of one call, 0 for sizes beyond the limits."""
    return int(_C.lib().bevb200_transfusion_proposals_workspace_bytes(B, C, H, W))


def _validate(x, K, k, exempt):
    if not isinstance(x, torch.Tensor):
        raise TypeError("dense_heatmap must be a torch.Tensor")
    if x.dim() != 4:
        raise ValueError("dense_heatmap must be [B, C, H, W], got %s" % (tuple(x.shape),))
    B, C, H, W = x.shape
    if min(B, C, H, W) < 1:
        raise ValueError("empty dense_heatmap %s" % (tuple(x.shape),))
    if k < 3 or k % 2 == 0:
        raise ValueError("nms_kernel_size must be odd and at least 3 (got %d)" % k)
    if H < k or W < k:
        raise ValueError("the %d x %d map is smaller than nms_kernel_size %d" % (H, W, k))
    if any(c >= C for c in exempt):
        raise ValueError("the exempt classes %s need more than %d classes" % (exempt, C))
    if K < 1 or K > C * H * W:
        raise ValueError("num_proposals must be in 1..C * H * W = %d (got %d)" % (C * H * W, K))
    if B > MAX_BATCH or C > MAX_CLASSES or C * H * W > MAX_CELLS or K > MAX_PROPOSALS or k > MAX_KERNEL:
        raise ValueError("at most %d samples, %d classes, %d cells per sample, %d proposals and kernel %d "
                         "(got %s, num_proposals %d, nms_kernel_size %d)"
                         % (MAX_BATCH, MAX_CLASSES, MAX_CELLS, MAX_PROPOSALS, MAX_KERNEL, (B, C, H, W), K, k))
    if x.dtype not in _DTYPES:
        raise ValueError("dense_heatmap must be fp32 or fp16, got %s" % x.dtype)
    if not x.is_cuda:
        raise ValueError("dense_heatmap must be a CUDA tensor: bevfusion_b200 has no CPU implementation")


def transfusion_proposals(dense_heatmap, num_proposals, nms_kernel_size=3, dataset="nuScenes"):
    """TransFusionHead's query selection from dense_heatmap [B, C, H, W] logits (fp32 or fp16, CUDA): returns
    (labels [B, K] int64 = flat // (H * W), index [B, K] int64 = flat % (H * W), query_heatmap_score [B, C, K] =
    the masked heatmap at every class of each selected cell, in the heatmap's dtype), K = num_proposals.
    Raises ValueError for an even or unit nms_kernel_size, a map smaller than the kernel, an exempt class >= C,
    K outside 1..C * H * W, another dtype, a CPU tensor or sizes beyond the module's MAX_* limits."""
    K, k = int(num_proposals), int(nms_kernel_size)
    exempt = exempt_classes(dataset)
    _validate(dense_heatmap, K, k, exempt)
    x = dense_heatmap.detach().contiguous()
    B, C, H, W = x.shape
    dev = x.device
    labels = torch.empty((B, K), dtype=torch.int64, device=dev)
    index = torch.empty((B, K), dtype=torch.int64, device=dev)
    score = torch.empty((B, C, K), dtype=x.dtype, device=dev)
    ws_bytes = workspace_bytes(B, C, H, W)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    ex = list(exempt) + [-1] * (2 - len(exempt))
    with torch.cuda.device(dev):
        _C.check(_C.lib().bevb200_transfusion_proposals(
            _C.ptr(x), _DTYPES[x.dtype], B, C, H, W, K, k, ex[0], ex[1], _C.ptr(labels), _C.ptr(index),
            _C.ptr(score), _C.ptr(ws), ws_bytes, _C.current_stream(dev)), "transfusion_proposals")
    return labels, index, score
