"""ctypes loader for libiggt_b200.so (the C-ABI in include/iggt_b200.h).

The product path has no CPU or PyTorch fallback: if the shared library is missing or a launcher
returns a non-zero status, a RuntimeError is raised.
"""
import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("IGGT_B200_LIB") or os.path.join(_HERE, "lib", "libiggt_b200.so")   # override: dev builds
CSRC_DIR = os.path.join(_HERE, "csrc")

_lib = None

c_void_p, c_int, c_int64, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float

# name -> argtypes ; every function returns int except iggt_version
SIGNATURES = {
    "iggt_device_info": [ctypes.POINTER(c_int), ctypes.POINTER(c_int)],
    "iggt_gemm_store16": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int,
                          c_void_p, c_int, c_void_p, c_int, c_int64, c_void_p],
    "iggt_gemm_resid32": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int,
                          c_void_p, c_void_p, c_int, c_void_p],
    "iggt_gemm_store32": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int,
                          c_void_p, c_int, c_void_p],
    "iggt_gemm_qkv": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int,
                      c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                      c_int, c_void_p, c_int, c_int, c_void_p],
    "iggt_kv_gather_maps": [c_void_p, c_int, c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p],
    "iggt_conv_nhwc": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                       c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p],
    "iggt_attention_fwd": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64,
                           c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p],
    "iggt_attention_plan": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "iggt_attention_fwd_ws": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64,
                              c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_int, c_void_p, c_int64, c_void_p],
    "iggt_attention_schedule_splits": [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p],
    "iggt_layernorm": [c_void_p, c_int64, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_int64,
                       c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_patchify": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_dino_assemble": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                           c_void_p],
    "iggt_upsample_bilinear_nhwc": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                    c_void_p, c_int, c_void_p],
    "iggt_deconv_shuffle": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_im2col3x3_s2": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_dpt_tail_fused": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                            c_int, c_int, c_int, c_int, c_void_p],
    "iggt_skinny_gemm": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                         c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_small_attention": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p],
    "iggt_token_attention": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p],
    "iggt_camera_head_workspace": [c_int],
    "iggt_camera_head": [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_layernorm16": [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_int, c_void_p],
    "iggt_col2im_k4s2p1": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_ocab_attention": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                            c_void_p],
    "iggt_window_attention": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_channel_mean": [c_void_p, c_void_p, c_int, c_int64, c_int, c_int, c_void_p],
    "iggt_se_scale_add": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                          c_int64, c_int, c_int, c_float, c_int, c_void_p],
    "iggt_pose_to_cameras": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "iggt_unproject_depth": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_float,
                             c_void_p],
    "iggt_resample_h_u8": [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p],
    "iggt_resample_v_u8_f32": [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int64,
                               c_int64, c_void_p],
    "iggt_knn_morton": [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p],
    "iggt_knn_reorder": [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p],
    "iggt_knn_mean_features": [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_void_p],
    "iggt_cluster_morton": [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p],
    "iggt_cluster_reorder": [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p],
    "iggt_cluster_core": [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p],
    "iggt_cluster_mst_workspace": [c_int64, ctypes.POINTER(c_int64)],
    "iggt_cluster_mst": [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                         ctypes.POINTER(ctypes.c_int32), c_void_p],
    "iggt_cluster_fill": [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                          c_void_p],
    "iggt_hdbscan_labels": [c_void_p, c_int64, c_int64, ctypes.c_double, c_void_p],
    "iggt_mst_orient": [c_void_p, c_int64, c_int64],
    "iggt_pca_basis_workspace": [c_int, ctypes.POINTER(c_int64)],
    "iggt_pca_basis": [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                       c_void_p],
    "iggt_pca_project": [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_int64, c_void_p],
    "iggt_quantile_workspace": [c_int64, ctypes.POINTER(c_int64)],
    "iggt_quantile": [c_void_p, c_int64, c_int64, c_int64, ctypes.POINTER(c_float), c_int, c_void_p, c_void_p,
                      c_void_p],
    "iggt_pca_stretch": [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p],
    "iggt_sym_eig": [c_void_p, c_int, c_void_p, c_void_p],
    "iggt_select": [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int, ctypes.POINTER(c_float), c_int,
                    c_void_p, c_void_p, c_void_p, c_void_p],
    "iggt_quantile_rule": [c_void_p, c_int64, c_int, c_float, ctypes.POINTER(c_float)],
    "iggt_resize_nearest": [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p],
    "iggt_zoom_nearest_index": [c_int, c_int, c_void_p],
    "iggt_depth_valid_mask": [c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p, c_void_p],
    "iggt_depth_metrics_workspace": [c_int64, ctypes.POINTER(c_int64)],
    "iggt_depth_metrics": [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p, c_int, c_float, c_float,
                           c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "iggt_pose_errors": [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p],
    "iggt_pose_errors_host": [c_void_p, c_void_p, c_int, c_void_p, c_void_p],
    "iggt_depth_zero_outside": [c_void_p, c_int64, c_int64, c_void_p, c_int, c_int, c_float, c_void_p],
    "iggt_depth_to_cam": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "iggt_pointcloud_workspace": [c_int64, ctypes.POINTER(c_int64)],
    "iggt_pointcloud_select": [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int64, c_int64, c_int64,
                               c_int64, c_int, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p],
    "iggt_pointcloud_compact": [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p],
    "iggt_mask_overlaps": [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                           c_void_p, c_void_p],
    "iggt_linear_sum_assignment": [c_void_p, c_int64, c_int64, c_void_p, c_void_p],
    "iggt_avgpool2_nhwc": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_sample_bilinear_nhwc": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "iggt_corr_sample": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                         c_void_p],
    "iggt_track_input": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                         c_int, c_int, c_int, c_float, c_int, c_void_p],
    "iggt_layernorm_rows": [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_int64, c_void_p, c_void_p, c_int,
                            c_int, c_void_p],
    "iggt_gemm_plan": [c_int, c_int, c_int, c_int, c_void_p],
    "iggt_attention_schedule": [c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int],
    "iggt_special_tokens": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
}


class CameraBlock(ctypes.Structure):
    """iggt_camera_block (include/iggt_b200.h)"""
    _fields_ = [(n, c_void_p) for n in ("n1w", "n1b", "qkv_w", "qkv_b", "proj_w", "proj_b", "ls1", "n2w", "n2b", "fc1_w",
                                        "fc1_b", "fc2_w", "fc2_b", "ls2")]


class CameraWeights(ctypes.Structure):
    """iggt_camera_weights (include/iggt_b200.h)"""
    _fields_ = ([(n, c_void_p) for n in ("emb_w", "emb_b", "mod_w", "mod_b")] + [("blk", CameraBlock * 4)] +
                [(n, c_void_p) for n in ("tok_w", "tok_b", "trk_w", "trk_b", "pb1_w", "pb1_b", "pb2_w", "pb2_b", "empty")])


def build(verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC_DIR, "-j", str(min(16, os.cpu_count() or 4))]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("building libiggt_b200.so failed:\n" + res.stdout[-4000:] + res.stderr[-4000:])
    if verbose:
        print(res.stdout[-2000:])
    return LIB_PATH


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the IGGT hot path)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.argtypes = argtypes
        fn.restype = c_int
    lib.iggt_version.restype = ctypes.c_char_p
    lib.iggt_version.argtypes = []
    lib.iggt_camera_head_workspace.restype = c_int64
    _lib = lib
    return lib


def check(status: int, what: str):
    if status != 0:
        raise RuntimeError(f"{what} failed with status {status} "
                           f"({'argument/setup error' if status < 0 else 'cudaError_t'})")
