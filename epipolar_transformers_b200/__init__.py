"""H100-native (sm_90a) epipolar-transformer fusion path (drop-in for the reference's
modeling/layers/epipolar.py::Epipolar + the projection helpers of vision/multiview.py).

    from epipolar_transformers_b200 import Epipolar, set_global_cfg
    sampler = Epipolar()                       # reads the global cfg like the reference
    out, corr_pos, attn, locs = sampler(feat_ref, feat_src, KRT_ref, KRT_src)

The arithmetic runs in libepipolar_b200.so (hand-written sm_90a CUDA behind the C ABI in
include/epipolar_b200.h).  Importing this package does not need a GPU; calling the op does,
and fails loudly if the library is missing.
"""
from .config import Node, default_cfg, make_cfg, get_global_cfg, set_global_cfg, cfg_h36m_r50_256, cfg_h36m_r152_384
from .epipolar import (Epipolar, FusionState, ZeroInitBN, epipolar_fusion, epipolar_fusion_multi, epipolar_fusion_views,
                       epipolar_fusion_views_backward, fold_z_bn, fold_head, head_weights, sample_locs, fused_other_feat, multitest, multitest_views, standard_views_test, view_source_table)
from .host_pipeline import HostStreamer, bind_host_to_gpu
from .peaks import find_tensor_peak_batch, find_tensor_peak_best
from .triangulate import triangulate_views
from .rpsm import H36M_PARENTS, crop_affine, limb_lengths, rpsm_pairwise, rpsm_views
from . import multiview, synthetic

__all__ = ["Epipolar", "FusionState", "HostStreamer", "bind_host_to_gpu", "ZeroInitBN", "epipolar_fusion", "fold_z_bn", "fold_head", "head_weights", "sample_locs", "fused_other_feat", "find_tensor_peak_batch",
           "epipolar_fusion_multi", "multitest", "find_tensor_peak_best", "epipolar_fusion_views", "epipolar_fusion_views_backward", "multitest_views",
           "standard_views_test", "view_source_table", "triangulate_views",
           "rpsm_views", "rpsm_pairwise", "limb_lengths", "crop_affine", "H36M_PARENTS",
           "Node", "default_cfg", "make_cfg", "get_global_cfg", "set_global_cfg",
           "cfg_h36m_r50_256", "cfg_h36m_r152_384", "multiview", "synthetic"]
