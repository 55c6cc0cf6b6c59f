"""ctypes binding of libcatgrasp_b200.so (the C ABI declared in include/catgrasp_b200.h).

The product path has NO CPU fallback: if the shared library is missing or no
H100 is present, every entry point raises.  Build the library with
``python -c "import __graft_entry__ as g; g.build()"`` (nvcc, sm_90a).

``SIGNATURES`` records, per entry point, which pointer parameters are read on the host (``HostBuf``) and which on the
device (``DevBuf``), and on which stream the call runs.  ``Context.call`` checks the arguments against it before any
launch, so a host address never reaches a kernel.

The package's functions follow one rule for their inputs and results: numpy in, numpy out; a CUDA tensor in, CUDA
tensors out on that tensor's device (``inputs`` and ``returned``).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libcatgrasp_b200.so")

CG_OK, CG_EINVAL, CG_ECUDA, CG_ENOMEM, CG_EUNSUPPORTED = 0, -1, -2, -3, -4
CG_NET_CLS, CG_NET_SEG = 0, 1
CG_SDF_TRILINEAR, CG_SDF_NEAREST = 0, 1
CG_ST_ACCEPT, CG_ST_REJ_DIR, CG_ST_REJ_IK, CG_ST_REJ_COLL, CG_ST_REJ_COLL_ENCL = 0, 1, 2, 3, 4


class CgError(RuntimeError):
    pass


class FilterParams(C.Structure):
    _fields_ = [
        ("nocs_pose", C.c_float * 16),
        ("canonical_to_nocs", C.c_float * 16),
        ("gripper_in_grasp", C.c_float * 16),
        ("filter_approach_dir_face_camera", C.c_int),
        ("adjust_collision_pose", C.c_int),
        ("sdf_mode", C.c_int),
        ("sdf_margin", C.c_float),
        ("split_coll_status", C.c_int),
    ]


class IkParams(C.Structure):
    _fields_ = [
        ("cam_in_world", C.c_float * 16),
        ("ee_in_grasp", C.c_float * 16),
        ("upper", C.c_double * 7),
        ("lower", C.c_double * 7),
    ]


class _Buffer:
    """ctypes argtype of a data pointer parameter.  ``from_param`` takes a contiguous torch tensor or numpy array of
    the parameter's kind, or anything ``c_void_p`` takes (None, a ``c_void_p`` from ``ptr``, ``byref``, an int
    address, a ctypes array) unchanged.  A non-contiguous buffer raises ValueError, one of the wrong kind TypeError."""
    on_device = None

    @classmethod
    def from_param(cls, a):
        if hasattr(a, "data_ptr"):
            if a.is_cuda != cls.on_device:
                raise TypeError(f"{cls.__name__} parameter got a tensor on {a.device}")
            if not a.is_contiguous():
                raise ValueError(f"{cls.__name__} parameter got a non-contiguous tensor of shape {tuple(a.shape)}")
            return C.c_void_p(a.data_ptr())
        if isinstance(a, np.ndarray):
            if cls.on_device:
                raise TypeError("DevBuf parameter got a numpy array")
            if not a.flags.c_contiguous:
                raise ValueError(f"HostBuf parameter got a non-contiguous array of shape {a.shape}")
            return C.c_void_p(a.ctypes.data)
        return C.c_void_p.from_param(a)


class HostBuf(_Buffer):
    """A pointer the library reads or writes on the host: numpy arrays and CPU tensors."""
    on_device = False


class DevBuf(_Buffer):
    """A pointer the library hands to a kernel: CUDA tensors."""
    on_device = True


_vp, _i, _f, _d, _sz, _H, _D = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t, HostBuf, DevBuf
# Stream an entry runs on when called through Context.call: TORCH = the current torch stream of the context's device
# (the entry works on the caller's device buffers), OWN = the context's own stream (the entry stages host data itself
# and synchronises), None = no switch (no stream work, or no context).
TORCH, OWN = "torch", "own"

# name -> (restype, argtypes, stream); must list every symbol of include/catgrasp_b200.h.  Handles (cg_ctx, cg_net,
# cg_sdf, cg_mlp, cg_cloud_index) and the CUDA stream are c_void_p; every other pointer is HostBuf or DevBuf.
SIGNATURES = {
    "cg_ctx_create": (_i, [_i, _H], None),
    "cg_ctx_destroy": (None, [_vp], None),
    "cg_ctx_set_stream": (_i, [_vp, _vp], None),
    "cg_ctx_use_own_stream": (_i, [_vp], None),
    "cg_ctx_synchronize": (_i, [_vp], None),
    "cg_last_error": (C.c_char_p, [_vp], None),
    "cg_version": (C.c_char_p, [], None),
    "cg_ctx_launch_count": (C.c_int64, [_vp], None),
    "cg_ctx_reset_launch_count": (None, [_vp], None),
    "cg_ctx_set_engine": (_i, [_vp, _i], None),
    "cg_ctx_get_engine": (_i, [_vp], None),
    "cg_ctx_fp16_overflow": (_i, [_vp, _H], None),
    "cg_ctx_profile": (_i, [_vp, _i], None),
    "cg_ctx_profile_read": (_i, [_vp, _H, _H], None),
    "cg_net_create": (_i, [_vp, _i, _i, _H, _sz, _H], OWN),
    "cg_net_destroy": (None, [_vp], None),
    "cg_net_blob_floats": (_sz, [_i, _i], None),
    "cg_graspq_forward_host": (_i, [_vp, _H, _H, _i, _H, _i, _H, _i, _H, _H, _H, _H], OWN),
    "cg_graspq_forward_dev": (_i, [_vp, _D, _D, _i, _D, _i, _D, _i, _D, _D, _D, _D], TORCH),
    "cg_graspq_forward_many_dev": (_i, [_vp, _D, _D, _i, _D, _i, _D, _i, _D, _D, _H, _i, _D, _D], TORCH),
    "cg_host_legacy_choice": (_i, [_H, _H, C.c_int64, C.c_int32, C.c_int32, _H, C.c_int32], None),
    "cg_host_legacy_skip": (_i, [_H, _H, C.c_int64, C.c_int32, C.c_int32], None),
    "cg_host_rng_isa": (_i, [_i], None),
    "cg_draw_ids_dev": (_i, [_vp, _i, _i, _i, C.c_uint64, C.c_int64, _D], TORCH),
    "cg_draw_ids_many_dev": (_i, [_vp, _i, _D, _D, _D, _D, _i, _i, _D], TORCH),
    "cg_mlp_create": (_i, [_vp, _i, _H, _H, _H, _H], OWN),
    "cg_mlp_destroy": (None, [_vp], None),
    "cg_shared_mlp_dev": (_i, [_vp, _D, C.c_int64, _D], TORCH),
    "cg_group_mlp_max_dev": (_i, [_vp, _D, _i, _i, _D], TORCH),
    "cg_three_interp_dev": (_i, [_vp, _D, _D, _D, _i, _D, _i, _i, _i, _i, _D, _D, _D], TORCH),
    "cg_cls_forward_dev": (_i, [_vp, _D, _i, _i, _D, _D], TORCH),
    "cg_seg_forward_dev": (_i, [_vp, _D, _i, _i, _D], TORCH),
    "cg_encoder_probe_dev": (_i, [_vp, _D, _D, _D, _i, _D, _D, _D, _D, _i, _i, _D, _D, _D, _D], TORCH),
    "cg_nunocs_forward_host": (_i, [_vp, _H, _i, _i, _H, _H, _H], OWN),
    "cg_nunocs_forward_dev": (_i, [_vp, _D, _i, _i, _D, _D, _D], TORCH),
    "cg_nunocs_forward_many_host": (_i, [_vp, _H, _i, _i, _i, _H, _H, _H], OWN),
    "cg_nunocs_forward_many_dev": (_i, [_vp, _D, _i, _i, _i, _D, _D, _D], TORCH),
    "cg_sdf_create": (_i, [_vp, _H, _i, _i, _i, _H, _f, _H], OWN),
    "cg_sdf_destroy": (None, [_vp], None),
    "cg_sdf_lookup_dev": (_i, [_vp, _D, _i, _i, _D], TORCH),
    "cg_sdf_from_mesh": (_i, [_vp, _H, _i, _H, _i, _f, _i, _H], OWN),
    "cg_sdf_geometry": (_i, [_vp, _H, _H, _H], None),
    "cg_sdf_download": (_i, [_vp, _H], OWN),
    "cg_filter_grasp_pose_host": (_i, [_vp, _H, _H, _i, _H, _i, _vp, _H, _i, _vp, _H, _i, _H, _H, _H], OWN),
    "cg_filter_grasp_pose_dev": (_i, [_vp, _H, _D, _i, _D, _i, _vp, _D, _i, _vp, _D, _i, _D, _D, _D], TORCH),
    "cg_iiwa14_ik_dev": (_i, [_vp, _D, _i, _H, _H, _D, _D], TORCH),
    "cg_filter_apply_ik_dev": (_i, [_vp, _H, _D, _i, _D, _i, _H, _D, _D, _D], TORCH),
    "cg_occupancy_grid_geometry": (_i, [_H, _i, _f, _H, _H], None),
    "cg_occupancy_from_scan_host": (_i, [_vp, _H, _i, _f, _H], OWN),
    "cg_ransac9d_host": (_i, [_vp, _H, _H, _i, _H, _i, _d, _H, _H, _H, _H, _H, _H], OWN),
    "cg_ransac9d_pose_dev": (_i, [_vp, _D, _D, _i, _D, _i, _H, _i, _H, _H, _H, _d, _D], TORCH),
    "cg_ransac9d_pose_many_dev": (_i, [_vp, _D, _D, _i, _i, _D, _i, _H, _i, _H, _H, _H, _d, _D], TORCH),
    "cg_ransac9d_kdtree_host": (_i, [_vp, _H, _H, _i, _H, _i, _d, _H, _H, _H, _d, _H, _H, _H], OWN),
    "cg_ransac9d_kdtree_pose_dev": (_i, [_vp, _D, _D, _i, _D, _i, _H, _i, _H, _H, _H, _d, _d, _D], TORCH),
    "cg_cone_poses_dev": (_i, [_vp, _D, _D, _i, _D, _i, _D, _i, _D, _i, _d, _D, _D], TORCH),
    "cg_center_grasps_dev": (_i, [_vp, _D, _D, _i, _D, _i], TORCH),
    "cg_grasp_affordance_dev": (_i, [_vp, _D, _i, _D, _D, _D, _i, _H, _H, _i, _d, _D, _D], TORCH),
    "cg_depth2xyz_dev": (_i, [_vp, _D, _i, _i, _i, _H, _D], TORCH),
    "cg_cloud_index_create": (_i, [_vp, _D, _i, _d, _H], TORCH),
    "cg_cloud_index_destroy": (None, [_vp], None),
    "cg_cloud_index_info": (_i, [_vp, _H, _H, _H, _H], None),
    "cg_voxel_down_sample_dev": (_i, [_vp, _D, _D, _D], TORCH),
    "cg_cloud_nearest_dev": (_i, [_vp, _D, _i, _d, _D, _D], TORCH),
    "cg_cloud_radius_mask_dev": (_i, [_vp, _D, _i, _d, _i, _D], TORCH),
    "cg_cloud_normals_dev": (_i, [_vp, _d, _i, _H, _D, _D, _D], TORCH),
    "cg_meanshift_dev": (_i, [_vp, _D, _i, _d, _i, _D, _D, _D, _D, _D], TORCH),
    "cg_spconv_index_dev": (_i, [_vp, _D, _i, _D, _D, _D, _D], TORCH),
    "cg_spconv_down_dev": (_i, [_vp, _D, _D, _i, _H, _i, _D, _D, _D, _D, _D], TORCH),
    "cg_spconv_index_many_dev": (_i, [_vp, _D, _i, _i, _H, _H, _D, _D, _D, _D, _D], TORCH),
    "cg_spconv_down_many_dev": (_i, [_vp, _D, _D, _D, _i, _i, _H, _i, _D, _D, _D, _D, _D, _D], TORCH),
    "cg_spconv_conv_dev": (_i, [_vp, _D, _i, _D, _i, _D, _i, _D, _i, _D, _D, _D, _D, _D], TORCH),
    "cg_pointgroup_voxel_mean_dev": (_i, [_vp, _D, _i, _i, _D, _D, _i, _D], TORCH),
    "cg_pointgroup_head_dev": (_i, [_vp, _D, _i, _D, _i, _D, _D, _D, _D, _D, _D, _D, _i, _D, _D], TORCH),
    "cg_segment_table_dev": (_i, [_vp, _D, _i, _D, _i, _i, _i, _D, _D, _D, _D, _D, _D, _D, _D, _D], TORCH),
    "cg_rank_grasps_dev": (_i, [_vp, _D, _i, _i, _i, _D, _D, _D, _D], TORCH),
    "cg_square_distance_dev": (_i, [_vp, _D, _D, _i, _i, _i, _D], TORCH),
    "cg_index_points_dev": (_i, [_vp, _D, _D, _i, _i, _i, _i, _D], TORCH),
    "cg_fps_dev": (_i, [_vp, _D, _i, _i, _i, _D, _D], TORCH),
    "cg_fps_single_cta_dev": (_i, [_vp, _D, _i, _i, _i, _D, _D], TORCH),
    "cg_ball_query_dev": (_i, [_vp, _f, _i, _D, _D, _i, _i, _i, _D], TORCH),
    "cg_group_points_dev": (_i, [_vp, _D, _D, _D, _D, _i, _i, _i, _i, _i, _D], TORCH),
}

_lib = None


def load():
    """Load the shared library (once) and attach prototypes.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CgError(
            f"{LIB_PATH} is missing: the CUDA extension has not been built "
            "(run __graft_entry__.build()). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args, _) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here means header/library drift
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def ptr(t):
    """Device/host pointer of a torch tensor or numpy array (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return C.c_void_p(t.data_ptr())
    return C.c_void_p(t.ctypes.data)


class Context:
    """One library context per device (stream + workspaces)."""

    _per_device = {}

    def __init__(self, device=0):
        lib = load()
        self.lib = lib
        self.device = int(device)
        h = _vp()
        rc = lib.cg_ctx_create(self.device, C.byref(h))
        if rc != CG_OK:
            raise CgError(f"cg_ctx_create(device={device}) failed with {rc}: "
                          "an H100 (sm_90) GPU is required; there is no CPU fallback")
        self.h = h

    @classmethod
    def get(cls, device=None):
        import torch
        if device is None:
            device = torch.cuda.current_device() if torch.cuda.is_available() else 0
        device = int(device)
        if device not in cls._per_device:
            cls._per_device[device] = cls(device)
        return cls._per_device[device]

    def check(self, rc):
        if rc != CG_OK:
            msg = self.lib.cg_last_error(self.h)
            raise CgError(f"libcatgrasp_b200 error {rc}: {msg.decode() if msg else ''}")

    def call(self, name, *args):
        """Call entry point ``name`` with ``args`` in header order, on this context: the context that created the
        handle the entry takes, if it takes one.  Every pointer argument is checked against its parameter
        (``HostBuf`` / ``DevBuf``) and every CUDA tensor must be on this context's device, all before the context
        switches to the entry's stream and calls it.  A non-zero status raises CgError; other results are returned."""
        res, argtypes, stream = SIGNATURES[name]
        conv = list(args)      # `args` keeps the buffers alive until the call returns
        for i, t in enumerate(argtypes):
            if t is HostBuf or t is DevBuf:
                a = args[i]
                if getattr(a, "is_cuda", False) and a.device.index != self.device:
                    raise CgError(f"{name}: argument {i + 1} is on {a.device}, the context on cuda:{self.device}")
                conv[i] = t.from_param(a)
        if stream is TORCH:
            self.use_torch_stream()
        elif stream is OWN:
            self.use_own_stream()
        rc = getattr(self.lib, name)(*conv)
        if res is _i:
            self.check(rc)
        return rc

    def use_torch_stream(self):
        import torch
        s = torch.cuda.current_stream(self.device).cuda_stream
        self.check(self.lib.cg_ctx_set_stream(self.h, C.c_void_p(s)))

    def use_own_stream(self):
        self.check(self.lib.cg_ctx_use_own_stream(self.h))

    def synchronize(self):
        self.check(self.lib.cg_ctx_synchronize(self.h))

    def set_engine(self, engine):
        self.check(self.lib.cg_ctx_set_engine(self.h, int(engine)))

    def get_engine(self):
        return int(self.lib.cg_ctx_get_engine(self.h))

    def fp16_overflow(self):
        """True if engine 2/3 had to clamp an activation to the fp16 range since the last call (clears the flag)."""
        v = C.c_int()
        self.check(self.lib.cg_ctx_fp16_overflow(self.h, C.byref(v)))
        return bool(v.value)

    def profile(self, enable):
        self.check(self.lib.cg_ctx_profile(self.h, int(bool(enable))))

    def profile_read(self):
        ms, n = C.c_double(), C.c_int64()
        self.check(self.lib.cg_ctx_profile_read(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def launch_count(self):
        return int(self.lib.cg_ctx_launch_count(self.h))

    def reset_launch_count(self):
        self.lib.cg_ctx_reset_launch_count(self.h)


def inputs(*arrays, dtype, ctx=None):
    """``(ctx, *tensors)``: ``ctx``, else the context of the first CUDA tensor's device, else the current device's;
    and every array (numpy, tensor, nested list; None stays None) as a contiguous tensor on that device, of ``dtype``
    (one torch dtype for all, or a tuple of one per array)."""
    import torch
    if ctx is None:
        ctx = Context.get(next((a.device.index for a in arrays if isinstance(a, torch.Tensor) and a.is_cuda), None))
    dev = torch.device("cuda", ctx.device)
    dtypes = dtype if isinstance(dtype, tuple) else (dtype,) * len(arrays)
    return (ctx, *[None if a is None else (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a)))
                   .to(device=dev, dtype=t).contiguous() for a, t in zip(arrays, dtypes)])


def returned(like, *results):
    """The results (CUDA tensors) as they are when ``like`` is a CUDA tensor, else as numpy arrays; one result comes
    back bare, several as a tuple."""
    if not getattr(like, "is_cuda", False):
        results = tuple(r.cpu().numpy() for r in results)
    return results[0] if len(results) == 1 else results
