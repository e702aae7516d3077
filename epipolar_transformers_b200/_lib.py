"""ctypes binding of libepipolar_b200.so (the C ABI in include/epipolar_b200.h).

There is NO fallback: if the CUDA library is missing or does not export the ABI the import of
the op fails loudly (RuntimeError), so a GPU box can never silently run another code path.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libepipolar_b200.so")

EPI_ABI_VERSION = 3
EPI_DTYPE_F32, EPI_DTYPE_BF16, EPI_DTYPE_F16 = 0, 1, 2
EPI_DTYPE_F64 = 3                   # the cameras of epi_triangulate_dlt_f64 only


def EPI_OUT_DTYPE(d):
    """`out`'s element type in bits 8-15 of EpiFusionParams.feat_dtype (include/epipolar_b200.h): maps | EPI_OUT_DTYPE(out)"""
    return d << 8


EPI_VIEW_SOURCES_MAX = 256          # V·S entries of a source table (include/epipolar_b200.h)
EPI_VARIANT_AUTO, EPI_VARIANT_WARP, EPI_VARIANT_TILE, EPI_VARIANT_SECTOR, EPI_VARIANT_PIPE = 0, 1, 2, 3, 4
VARIANTS = {"auto": EPI_VARIANT_AUTO, "warp": EPI_VARIANT_WARP, "tile": EPI_VARIANT_TILE, "sector": EPI_VARIANT_SECTOR,
            "pipe": EPI_VARIANT_PIPE}

EXPORTS = ("epi_version", "epi_last_error", "epi_fusion_workspace_bytes", "epi_fusion_cache_bytes", "epi_fusion_forward_f32",
           "epi_fusion_backward_workspace_bytes", "epi_fusion_backward_f32", "epi_find_peaks_f32", "epi_find_peaks_best_f32",
           "epi_sample_locs_f32", "epi_fold_z_bn_f32", "epi_last_launch_count", "epi_umma_selftest",
           "epi_kernel_timing_enable", "epi_kernel_timing_last_ms", "epi_kernel_timing_last3",
           "epi_fusion_backward_deterministic", "epi_fusion_views", "epi_fusion_view_sources_forward_f32",
           "epi_fusion_view_sources_workspace_bytes", "epi_fusion_view_sources_cache_bytes", "epi_fusion_view_sources",
           "epi_fusion_views_backward_f32", "epi_fusion_views_backward_workspace_bytes", "epi_fusion_views_backward",
           "epi_fold_head_f32", "epi_fusion_heatmaps_f32", "epi_fusion_heatmaps_workspace_bytes", "epi_fusion_heatmaps_cache_bytes",
           "epi_fusion_heatmaps", "epi_triangulate_dlt_f64", "epi_triangulate", "epi_rpsm_f32", "epi_rpsm_workspace_bytes",
           "epi_rpsm_pairwise_pack", "epi_rpsm")
# The source-table entry points are new symbols, not a reinterpreted field, so a library without them still runs every other
# form correctly: load() accepts it, and only a call with a source table needs them (`require_view_sources`).
VIEW_SOURCES_EXPORTS = ("epi_fusion_view_sources_forward_f32", "epi_fusion_view_sources_workspace_bytes",
                        "epi_fusion_view_sources_cache_bytes", "epi_fusion_view_sources")
# The backward of the views form is optional in the same way: only a views-backward call needs it (`require_views_backward`).
VIEWS_BACKWARD_EXPORTS = ("epi_fusion_views_backward_f32", "epi_fusion_views_backward_workspace_bytes", "epi_fusion_views_backward")
# So are the heat-map forward and its fold: only a call with a head needs them (`require_heatmaps`).
HEATMAPS_EXPORTS = ("epi_fold_head_f32", "epi_fusion_heatmaps_f32", "epi_fusion_heatmaps_workspace_bytes",
                    "epi_fusion_heatmaps_cache_bytes", "epi_fusion_heatmaps")
# And the triangulation: only `triangulate_views` needs it (`require_triangulate`).
TRIANGULATE_EXPORTS = ("epi_triangulate_dlt_f64", "epi_triangulate")
TRIANGULATE_MAX_VIEWS = 64          # epi_triangulate_dlt_f64's V (include/epipolar_b200.h)
# And the recursive pictorial structure: only `rpsm_views` and `rpsm_pairwise` need it (`require_rpsm`).
RPSM_EXPORTS = ("epi_rpsm_f32", "epi_rpsm_workspace_bytes", "epi_rpsm_pairwise_pack", "epi_rpsm")
RPSM_MAX_VIEWS, RPSM_MAX_JOINTS, RPSM_MAX_NBINS, RPSM_MAX_RECUR_NBINS, RPSM_MAX_DEPTH = 64, 32, 16, 4, 32
HEAD_MAX_JOINTS = 64                # EpiHeadParams.J (include/epipolar_b200.h)
PEAKS_MAX_R = 23169                 # EPI_PEAKS_MAX_R: the largest R = int(radius + 0.5) of the peak finders (include/epipolar_b200.h)

_fp = ctypes.POINTER(ctypes.c_float)


class EpiFusionParams(ctypes.Structure):
    """Field-for-field mirror of `struct EpiFusionParams` (include/epipolar_b200.h)."""
    _fields_ = [
        ("feat_ref", ctypes.c_void_p), ("ref_stride", ctypes.c_int64 * 4),
        ("feat_src", ctypes.c_void_p), ("src_stride", ctypes.c_int64 * 4),
        ("P_ref", ctypes.c_void_p), ("P_src", ctypes.c_void_p), ("sample_locs_in", ctypes.c_void_p),
        ("out", ctypes.c_void_p), ("out_stride", ctypes.c_int64 * 4),
        ("attn", ctypes.c_void_p), ("corr_pos", ctypes.c_void_p), ("sample_locs_out", ctypes.c_void_p),
        ("z_weight_folded", ctypes.c_void_p), ("z_bias_folded", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
        ("N", ctypes.c_int32), ("C", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32), ("K", ctypes.c_int32),
        ("downsample", ctypes.c_float), ("img_scale", ctypes.c_float), ("eps", ctypes.c_float), ("softmax_scale", ctypes.c_float),
        ("align_corners", ctypes.c_int32), ("correct_normalize", ctypes.c_int32), ("z_residual", ctypes.c_int32),
        ("add_ref_residual", ctypes.c_int32), ("variant", ctypes.c_int32), ("feat_dtype", ctypes.c_int32),
        ("n_src", ctypes.c_int32), ("reserved", ctypes.c_int32 * 1),
        ("cache", ctypes.c_void_p), ("cache_bytes", ctypes.c_size_t),
    ]

    # n_views shares its word with reserved[0] (an anonymous union in the header keeps the old name)
    @property
    def n_views(self):
        return self.reserved[0]

    @n_views.setter
    def n_views(self, v):
        self.reserved[0] = v


class EpiHeadParams(ctypes.Structure):
    """Field-for-field mirror of `struct EpiHeadParams` (include/epipolar_b200.h)."""
    _fields_ = [
        ("A", ctypes.c_void_p), ("B", ctypes.c_void_p), ("b", ctypes.c_void_p),
        ("heat", ctypes.c_void_p), ("heat_stride", ctypes.c_int64 * 4),
        ("J", ctypes.c_int32), ("reserved", ctypes.c_int32 * 3),
    ]


class EpiFusionBwdParams(ctypes.Structure):
    """Field-for-field mirror of `struct EpiFusionBwdParams` (include/epipolar_b200.h)."""
    _fields_ = [
        ("feat_ref", ctypes.c_void_p), ("ref_stride", ctypes.c_int64 * 4),
        ("feat_src", ctypes.c_void_p), ("src_stride", ctypes.c_int64 * 4),
        ("P_ref", ctypes.c_void_p), ("P_src", ctypes.c_void_p), ("sample_locs_in", ctypes.c_void_p),
        ("attn", ctypes.c_void_p),
        ("grad_out", ctypes.c_void_p), ("gout_stride", ctypes.c_int64 * 4),
        ("grad_attn", ctypes.c_void_p),
        ("grad_ref", ctypes.c_void_p), ("gref_stride", ctypes.c_int64 * 4),
        ("grad_src", ctypes.c_void_p), ("gsrc_stride", ctypes.c_int64 * 4),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
        ("N", ctypes.c_int32), ("C", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32), ("K", ctypes.c_int32),
        ("downsample", ctypes.c_float), ("img_scale", ctypes.c_float), ("eps", ctypes.c_float), ("softmax_scale", ctypes.c_float),
        ("align_corners", ctypes.c_int32), ("correct_normalize", ctypes.c_int32),
        ("grad_keys", ctypes.c_int32), ("grad_vals", ctypes.c_int32), ("feat_dtype", ctypes.c_int32),
        ("deterministic", ctypes.c_int32), ("reserved", ctypes.c_int32 * 2),
    ]


class EpiRpsmParams(ctypes.Structure):
    """Field-for-field mirror of `struct EpiRpsmParams` (include/epipolar_b200.h)."""
    _fields_ = [
        ("heat", ctypes.c_void_p), ("P", ctypes.c_void_p), ("crop", ctypes.c_void_p), ("root", ctypes.c_void_p),
        ("limb_length", ctypes.c_void_p), ("pairwise", ctypes.c_void_p), ("parents", ctypes.POINTER(ctypes.c_int32)),
        ("pose", ctypes.c_void_p), ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
        ("V", ctypes.c_int32), ("N", ctypes.c_int32), ("J", ctypes.c_int32), ("h", ctypes.c_int32), ("w", ctypes.c_int32),
        ("first_nbins", ctypes.c_int32), ("recur_nbins", ctypes.c_int32), ("recur_depth", ctypes.c_int32),
        ("align_corners", ctypes.c_int32), ("image_size", ctypes.c_float * 2), ("grid_size", ctypes.c_double),
        ("tolerance", ctypes.c_double),
    ]


_lib = None


def load():
    """Load the shared library once; raise if it is absent or the ABI does not match."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "epipolar_transformers_b200: CUDA library %s is missing. Build it with "
            "`python -m epipolar_transformers_b200.build` (needs nvcc). There is no CPU/PyTorch fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    optional = VIEW_SOURCES_EXPORTS + VIEWS_BACKWARD_EXPORTS + HEATMAPS_EXPORTS + TRIANGULATE_EXPORTS + RPSM_EXPORTS
    missing = [s for s in EXPORTS if s not in optional and not hasattr(lib, s)]
    if missing:
        # e.g. a library built before EpiFusionBwdParams.deterministic or EpiFusionParams.n_views, which would ignore the field
        # (a views call would silently run as a one-source call)
        raise RuntimeError("libepipolar_b200.so does not export %s; rebuild it with "
                           "`python -m epipolar_transformers_b200.build --force`" % missing)
    lib.epi_version.restype = ctypes.c_int
    lib.epi_last_error.restype = ctypes.c_char_p
    lib.epi_last_launch_count.restype = ctypes.c_int
    lib.epi_fusion_workspace_bytes.restype = ctypes.c_size_t
    lib.epi_fusion_workspace_bytes.argtypes = [ctypes.POINTER(EpiFusionParams)]
    lib.epi_fusion_cache_bytes.restype = ctypes.c_size_t
    lib.epi_fusion_cache_bytes.argtypes = [ctypes.POINTER(EpiFusionParams)]
    lib.epi_fusion_forward_f32.restype = ctypes.c_int
    lib.epi_fusion_forward_f32.argtypes = [ctypes.POINTER(EpiFusionParams), ctypes.c_void_p]
    lib.epi_fusion_backward_workspace_bytes.restype = ctypes.c_size_t
    lib.epi_fusion_backward_workspace_bytes.argtypes = [ctypes.POINTER(EpiFusionBwdParams)]
    lib.epi_fusion_backward_f32.restype = ctypes.c_int
    lib.epi_fusion_backward_f32.argtypes = [ctypes.POINTER(EpiFusionBwdParams), ctypes.c_void_p]
    lib.epi_find_peaks_f32.restype = ctypes.c_int
    lib.epi_find_peaks_f32.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                       ctypes.c_int32, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int32, ctypes.c_void_p]
    lib.epi_find_peaks_best_f32.restype = ctypes.c_int
    lib.epi_find_peaks_best_f32.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int32] * 5 + \
        [ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int32, ctypes.c_void_p]
    lib.epi_sample_locs_f32.restype = ctypes.c_int
    lib.epi_sample_locs_f32.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                        ctypes.c_int32, ctypes.c_int32, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                        ctypes.c_int32, ctypes.c_void_p]
    lib.epi_fold_z_bn_f32.restype = ctypes.c_int
    lib.epi_fold_z_bn_f32.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_float, ctypes.c_int32, ctypes.c_void_p,
                                                             ctypes.c_void_p, ctypes.c_void_p]
    lib.epi_umma_selftest.restype = ctypes.c_int
    lib.epi_umma_selftest.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_int, ctypes.c_void_p]
    lib.epi_kernel_timing_enable.restype = ctypes.c_int
    lib.epi_kernel_timing_enable.argtypes = [ctypes.c_int]
    lib.epi_kernel_timing_last_ms.restype = ctypes.c_float
    lib.epi_kernel_timing_last3.restype = ctypes.c_int
    lib.epi_kernel_timing_last3.argtypes = [ctypes.POINTER(ctypes.c_float)]
    lib.epi_fusion_backward_deterministic.restype = ctypes.c_int
    lib.epi_fusion_views.restype = ctypes.c_int
    if all(hasattr(lib, s) for s in VIEW_SOURCES_EXPORTS):
        table = [ctypes.POINTER(EpiFusionParams), ctypes.POINTER(ctypes.c_int32), ctypes.c_int32]
        lib.epi_fusion_view_sources_forward_f32.restype = ctypes.c_int
        lib.epi_fusion_view_sources_forward_f32.argtypes = table + [ctypes.c_void_p]
        lib.epi_fusion_view_sources_workspace_bytes.restype = ctypes.c_size_t
        lib.epi_fusion_view_sources_workspace_bytes.argtypes = table
        lib.epi_fusion_view_sources_cache_bytes.restype = ctypes.c_size_t
        lib.epi_fusion_view_sources_cache_bytes.argtypes = table
        lib.epi_fusion_view_sources.restype = ctypes.c_int
    if all(hasattr(lib, s) for s in VIEWS_BACKWARD_EXPORTS):
        views = [ctypes.POINTER(EpiFusionBwdParams), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32), ctypes.c_int32]
        lib.epi_fusion_views_backward_f32.restype = ctypes.c_int
        lib.epi_fusion_views_backward_f32.argtypes = views + [ctypes.c_void_p]
        lib.epi_fusion_views_backward_workspace_bytes.restype = ctypes.c_size_t
        lib.epi_fusion_views_backward_workspace_bytes.argtypes = views
        lib.epi_fusion_views_backward.restype = ctypes.c_int
    if all(hasattr(lib, s) for s in HEATMAPS_EXPORTS):
        heat = [ctypes.POINTER(EpiFusionParams), ctypes.POINTER(EpiHeadParams), ctypes.POINTER(ctypes.c_int32), ctypes.c_int32]
        lib.epi_fusion_heatmaps_f32.restype = ctypes.c_int
        lib.epi_fusion_heatmaps_f32.argtypes = heat + [ctypes.c_void_p]
        lib.epi_fusion_heatmaps_workspace_bytes.restype = ctypes.c_size_t
        lib.epi_fusion_heatmaps_workspace_bytes.argtypes = heat
        lib.epi_fusion_heatmaps_cache_bytes.restype = ctypes.c_size_t
        lib.epi_fusion_heatmaps_cache_bytes.argtypes = heat
        lib.epi_fusion_heatmaps.restype = ctypes.c_int
        lib.epi_fold_head_f32.restype = ctypes.c_int
        lib.epi_fold_head_f32.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 3
    if all(hasattr(lib, s) for s in TRIANGULATE_EXPORTS):
        lib.epi_triangulate_dlt_f64.restype = ctypes.c_int
        lib.epi_triangulate_dlt_f64.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int32, ctypes.c_double] + [ctypes.c_int32] * 3 + \
            [ctypes.c_void_p] * 3
        lib.epi_triangulate.restype = ctypes.c_int
    if all(hasattr(lib, s) for s in RPSM_EXPORTS):
        lib.epi_rpsm_f32.restype = ctypes.c_int
        lib.epi_rpsm_f32.argtypes = [ctypes.POINTER(EpiRpsmParams), ctypes.c_void_p]
        lib.epi_rpsm_workspace_bytes.restype = ctypes.c_size_t
        lib.epi_rpsm_workspace_bytes.argtypes = [ctypes.POINTER(EpiRpsmParams)]
        lib.epi_rpsm_pairwise_pack.restype = ctypes.c_int
        lib.epi_rpsm_pairwise_pack.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_double,
                                               ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p]
        lib.epi_rpsm.restype = ctypes.c_int
    v = lib.epi_version()
    if v != EPI_ABI_VERSION:
        raise RuntimeError("libepipolar_b200.so ABI version %d != expected %d" % (v, EPI_ABI_VERSION))
    _lib = lib
    return lib


def require_view_sources(lib):
    """Raise unless `lib` has the source-table form of the views call (epi_fusion_view_sources())."""
    missing = [s for s in VIEW_SOURCES_EXPORTS if not hasattr(lib, s)]
    if missing or lib.epi_fusion_view_sources() != 1:
        raise RuntimeError("libepipolar_b200.so does not export %s, so it cannot fuse views with a source table; rebuild it with "
                           "`python -m epipolar_transformers_b200.build --force`" % (missing or ["epi_fusion_view_sources"]))


def require_views_backward(lib):
    """Raise unless `lib` has the backward of the views form (epi_fusion_views_backward())."""
    missing = [s for s in VIEWS_BACKWARD_EXPORTS if not hasattr(lib, s)]
    if missing or lib.epi_fusion_views_backward() != 1:
        raise RuntimeError("libepipolar_b200.so does not export %s, so it has no backward for the views form; rebuild it with "
                           "`python -m epipolar_transformers_b200.build --force`" % (missing or ["epi_fusion_views_backward"]))


def require_heatmaps(lib):
    """Raise unless `lib` has the heat-map forward (epi_fusion_heatmaps())."""
    missing = [s for s in HEATMAPS_EXPORTS if not hasattr(lib, s)]
    if missing or lib.epi_fusion_heatmaps() != 1:
        raise RuntimeError("libepipolar_b200.so does not export %s, so it cannot run the pose head as the forward's epilogue; "
                           "rebuild it with `python -m epipolar_transformers_b200.build --force`" % (missing or ["epi_fusion_heatmaps"]))


def require_triangulate(lib):
    """Raise unless `lib` has the DLT triangulation (epi_triangulate())."""
    missing = [s for s in TRIANGULATE_EXPORTS if not hasattr(lib, s)]
    if missing or lib.epi_triangulate() != 1:
        raise RuntimeError("libepipolar_b200.so does not export %s, so it cannot triangulate joints; rebuild it with "
                           "`python -m epipolar_transformers_b200.build --force`" % (missing or ["epi_triangulate"]))


def require_rpsm(lib):
    """Raise unless `lib` has the recursive pictorial structure (epi_rpsm())."""
    missing = [s for s in RPSM_EXPORTS if not hasattr(lib, s)]
    if missing or lib.epi_rpsm() != 1:
        raise RuntimeError("libepipolar_b200.so does not export %s, so it cannot run the recursive pictorial structure; rebuild "
                           "it with `python -m epipolar_transformers_b200.build --force`" % (missing or ["epi_rpsm"]))


def check(rc: int, what: str):
    if rc != 0:
        msg = load().epi_last_error().decode("utf-8", "replace")
        raise RuntimeError("%s failed (code %d): %s" % (what, rc, msg))
