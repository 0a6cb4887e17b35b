"""ctypes binding of libvmap_b200.so (C ABI declared in include/vmap_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or fails to
load, every op raises.  ``build()`` compiles it in-tree with nvcc for sm_90a.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VMB_LIB") or os.path.join(_HERE, "libvmap_b200.so")   # VMB_LIB: another build of the library
CSRC = os.path.join(_HERE, "csrc")

VMB_IMPL = {"auto": 0, "fp32": 1, "umma": 2, "layerwise": 3}
VMB_ST_LOSS_EXPLODE = 1
VMB_ST_NONFINITE = 2
N_TENSORS = 15

_vp = C.c_void_p
_ll = C.c_longlong


class StepArgs(C.Structure):
    _fields_ = [
        ("n_obj", C.c_int), ("n_rays", C.c_int), ("n_samples", C.c_int), ("impl", C.c_int),
        ("pcs", _vp), ("pcs_stride", _ll),
        ("z_vals", _vp), ("z_stride", _ll),
        ("gt_depth", _vp), ("gt_depth_stride", _ll),
        ("gt_colour", _vp), ("gt_colour_stride", _ll),
        ("sem", _vp), ("sem_stride", _ll),
        ("mask_depth", _vp), ("mask_stride", _ll),
        ("params", _vp), ("image", _vp), ("scale", _vp), ("grads", _vp), ("loss_terms", _vp),
        ("r_depth", _vp), ("r_var", _vp), ("r_colour", _vp), ("r_opacity", _vp),
        ("counts", _vp),
        ("colour_scaling", C.c_float), ("opacity_scaling", C.c_float),
        ("backward", C.c_int), ("fuse_adam", C.c_int),
        ("k1_start_event", _vp), ("k1_stop_event", _vp),
        ("exp_avg", _vp), ("exp_avg_sq", _vp), ("step_counter", _vp), ("step", C.c_int),
        ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
        ("weight_decay", C.c_float), ("guard_loss", C.c_int), ("status", _vp), ("loss_sum", _vp),
    ]


class AdamArgs(C.Structure):
    _fields_ = [
        ("n_obj", C.c_int), ("step", C.c_int),
        ("params", _vp), ("grads", _vp), ("exp_avg", _vp), ("exp_avg_sq", _vp),
        ("image", _vp), ("loss_terms", _vp), ("status", _vp),
        ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
        ("weight_decay", C.c_float), ("zero_grads", C.c_int),
        ("step_counter", _vp), ("grad_scale", _vp),
    ]


class ForwardArgs(C.Structure):
    _fields_ = [
        ("n_obj", C.c_int), ("n_points", _ll),
        ("points", _vp), ("points_stride", _ll),
        ("params", _vp), ("scale", _vp),
        ("alpha", _vp), ("alpha_stride", _ll),
        ("colour", _vp), ("colour_stride", _ll),
        ("image", _vp),
    ]


class SampleArgs(C.Structure):
    _fields_ = [
        ("n_obj", C.c_int), ("n_frames", C.c_int), ("n_pix", C.c_int),
        ("n_bins_cam2surface", C.c_int), ("n_bins", C.c_int), ("width", C.c_int), ("height", C.c_int),
        ("min_bound", C.c_float), ("surface_eps", C.c_float), ("stop_eps", C.c_float),
        ("rgbs", _vp), ("depths", _vp), ("t_wc", _vp), ("bbox", _vp),
        ("n_keyframes", _vp), ("latest_kf", _vp), ("rays_dir", _vp), ("bin_limits", _vp),
        ("seed", C.c_ulonglong), ("offset", C.c_ulonglong),
        ("inj_kf", _vp), ("inj_u_w", _vp), ("inj_u_h", _vp), ("inj_u_z", _vp), ("inj_nrm", _vp),
        ("pcs", _vp), ("z_vals", _vp), ("gt_depth", _vp), ("gt_colour", _vp), ("gt_rgb_u8", _vp),
        ("sem", _vp), ("mask_depth", _vp),
        ("store_rgbx", _vp), ("store_depth", _vp), ("store_inst", _vp), ("store_t_wc", _vp),
        ("kf_slot", _vp), ("kf_bbox", _vp), ("obj_id", _vp), ("kf_stride", C.c_int),
        ("offset_dev", _vp),
    ]


class IngestArgs(C.Structure):
    _fields_ = [
        ("width", C.c_int), ("height", C.c_int), ("inst", _vp), ("cls", _vp), ("max_id", C.c_int),
        ("bbox_scale", C.c_float), ("min_extent", C.c_int), ("bg_class", _vp), ("n_class", C.c_int),
        ("stats", _vp), ("bbox", _vp), ("rgb", _vp), ("depth", _vp),
        ("dst_rgbx", _vp), ("dst_depth", _vp), ("dst_inst", _vp),
    ]


class McArgs(C.Structure):
    _fields_ = [
        ("volume", _vp), ("nx", C.c_int), ("ny", C.c_int), ("nz", C.c_int), ("level", C.c_float),
        ("affine", C.c_float * 12), ("totals", _vp),
        ("vertices", _vp), ("normals", _vp), ("faces", _vp), ("max_vertices", _ll), ("max_faces", _ll),
    ]


class UnprojectArgs(C.Structure):
    _fields_ = [
        ("width", C.c_int), ("height", C.c_int), ("n_keyframes", C.c_int),
        ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
        ("rgbs", _vp), ("depths", _vp), ("t_wc", _vp),
        ("store_depth", _vp), ("store_inst", _vp), ("store_t_wc", _vp), ("kf_slot", _vp), ("obj_id", C.c_int),
        ("count", _vp), ("points", _vp), ("max_points", _ll),
    ]


class ClipArgs(C.Structure):
    _fields_ = [
        ("vertices", _vp), ("n_vertices", _ll), ("faces", _vp), ("n_faces", _ll),
        ("center", C.c_float * 3), ("rotation", C.c_float * 9), ("extent", C.c_float * 3),
        ("count", _vp), ("triangles", _vp), ("max_triangles", _ll),
    ]


class SurfaceSampleArgs(C.Structure):
    _fields_ = [
        ("vertices", _vp), ("n_vertices", _ll), ("faces", _vp), ("n_faces", _ll),
        ("n_points", _ll), ("seed", C.c_ulonglong), ("uniforms", _vp), ("points", _vp), ("face_index", _vp),
    ]


class NnArgs(C.Structure):
    _fields_ = [
        ("ref", _vp), ("n_ref", _ll), ("query", _vp), ("n_query", _ll), ("dist", _vp), ("index", _vp),
    ]


EXPORTS = (
    "vmb_version", "vmb_param_count", "vmb_param_stride", "vmb_param_offsets", "vmb_image_bytes",
    "vmb_create", "vmb_destroy", "vmb_last_error", "vmb_step", "vmb_mask_counts", "vmb_adam",
    "vmb_build_image", "vmb_forward", "vmb_sample", "vmb_ingest_frame", "vmb_debug_gemm",
    "vmb_mc_count", "vmb_mc_emit", "vmb_unproject",
    "vmb_clip_count", "vmb_clip_emit", "vmb_surface_sample", "vmb_nn_dist",
)

_lib = None
_lock = threading.Lock()


class VmbError(RuntimeError):
    pass


def build(verbose: bool = False) -> str:
    """Compile libvmap_b200.so in-tree (nvcc, -gencode arch=compute_90a,code=sm_90a)."""
    r = subprocess.run(["make", "-C", CSRC], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout, r.stderr)
    if r.returncode != 0 or not os.path.isfile(LIB_PATH):
        raise VmbError("building libvmap_b200.so failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


def lib():
    """The loaded library; raises (never falls back) if it is not there."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise VmbError(f"{LIB_PATH} not found -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU / PyTorch fallback for the vMAP step)")
        L = C.CDLL(LIB_PATH)
        L.vmb_version.restype = C.c_char_p
        L.vmb_last_error.restype = C.c_char_p
        L.vmb_last_error.argtypes = [_vp]
        for n in ("vmb_param_count", "vmb_param_stride", "vmb_image_bytes"):
            getattr(L, n).argtypes = [C.c_int, C.c_int]
            getattr(L, n).restype = C.c_int
        L.vmb_param_offsets.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.vmb_create.argtypes = [C.POINTER(_vp), C.c_int, C.c_int, C.c_int, C.c_int]
        L.vmb_destroy.argtypes = [_vp]
        L.vmb_destroy.restype = None
        L.vmb_step.argtypes = [_vp, C.POINTER(StepArgs), _vp]
        L.vmb_adam.argtypes = [_vp, C.POINTER(AdamArgs), _vp]
        L.vmb_forward.argtypes = [_vp, C.POINTER(ForwardArgs), _vp]
        L.vmb_sample.argtypes = [_vp, C.POINTER(SampleArgs), _vp]
        L.vmb_ingest_frame.argtypes = [_vp, C.POINTER(IngestArgs), _vp]
        L.vmb_mc_count.argtypes = [_vp, C.POINTER(McArgs), _vp]
        L.vmb_mc_emit.argtypes = [_vp, C.POINTER(McArgs), _vp]
        L.vmb_unproject.argtypes = [_vp, C.POINTER(UnprojectArgs), _vp]
        L.vmb_clip_count.argtypes = [_vp, C.POINTER(ClipArgs), _vp]
        L.vmb_clip_emit.argtypes = [_vp, C.POINTER(ClipArgs), _vp]
        L.vmb_surface_sample.argtypes = [_vp, C.POINTER(SurfaceSampleArgs), _vp]
        L.vmb_nn_dist.argtypes = [_vp, C.POINTER(NnArgs), _vp]
        L.vmb_build_image.argtypes = [_vp, C.c_int, _vp, _vp, _vp]
        L.vmb_mask_counts.argtypes = [_vp, C.c_int, C.c_int, _vp, _ll, _vp, _ll, _vp, _vp]
        L.vmb_debug_gemm.argtypes = [C.c_int] * 7 + [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _vp, C.c_int, _vp, C.c_int,
                                     C.c_int, C.c_int, C.c_float, _vp]
        _lib = L
        return _lib


def check(handle, rc: int, what: str):
    if rc != 0:
        msg = lib().vmb_last_error(handle)
        raise VmbError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")


def param_layout(hidden: int, n_freq: int):
    """(count, stride, offsets[15], sizes[15]) of one object's row in the param block."""
    L = lib()
    off = (C.c_int * N_TENSORS)()
    sz = (C.c_int * N_TENSORS)()
    rc = L.vmb_param_offsets(hidden, n_freq, off, sz)
    if rc != 0:
        raise VmbError(f"vmb_param_offsets({hidden},{n_freq}) -> {rc}")
    return L.vmb_param_count(hidden, n_freq), L.vmb_param_stride(hidden, n_freq), list(off), list(sz)
