"""ctypes binding of the C ABI in include/dsm.h (the reference-facing boundary).

`FusionFunctions` mirrors the reference class of the same name (fusion_functions.h:23-95): the
same two public methods, same argument meaning.  It is a thin veneer: every call goes straight
into libdsm_b200.so; there is no Python or CPU implementation behind it, and loading fails
loudly when the library (or an H100) is missing.
"""
import ctypes
import os
import numpy as np

from .elements import POINT_DTYPE, SEED_DTYPE, SURFEL_DTYPE, num_seeds

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdsm_b200.so")

DSM_OK = 0
DSM_E_CAPACITY = -6  # a wait that returns it still carries its results (the map of the last applied frame)
ERRORS = {-1: "DSM_E_INVALID", -2: "DSM_E_SHAPE", -3: "DSM_E_NODEVICE", -4: "DSM_E_CUDA",
          -5: "DSM_E_NOMEM", -6: "DSM_E_CAPACITY", -7: "DSM_E_STATE", -8: "DSM_E_NCCL", -9: "DSM_E_IO"}
NUM_KERNELS = 10
WINDOW_MAX_KEYS = 128  # DSM_WINDOW_MAX_KEYS: keys per frame and list of dsm_fuse_stream_window

# every symbol include/dsm.h declares (tests/test_abi.py checks the library exports all of them)
EXPORTS = [
    "dsm_version", "dsm_strerror", "dsm_last_error", "dsm_create", "dsm_destroy", "dsm_num_seeds",
    "dsm_fuse_frame", "dsm_batch_upload", "dsm_batch_run", "dsm_batch_download", "dsm_sync",
    "dsm_fuse_batch", "dsm_fuse_batch_async", "dsm_batch_wait", "dsm_batch_restore_pool", "dsm_pool_upload", "dsm_fuse_frame_resident",
    "dsm_pool_transform", "dsm_pool_retire", "dsm_pool_append", "dsm_pool_size", "dsm_pool_download", "dsm_get_labels", "dsm_get_seeds",
    "dsm_debug_stop_after", "dsm_debug_invariant_violations", "dsm_profile_enable", "dsm_profile_reset", "dsm_profile_read", "dsm_kernel_name", "dsm_device_buffer",
    "dsm_pool_export_cloud", "dsm_pool_export_surfels", "dsm_write_pcd", "dsm_write_ply_mesh", "dsm_mesh_vertices", "dsm_fuse_stream_resident",
    "dsm_inactive_reserve", "dsm_inactive_retire", "dsm_inactive_reactivate", "dsm_inactive_transform", "dsm_inactive_export_cloud",
    "dsm_inactive_download", "dsm_inactive_size", "dsm_frame_raw_cloud", "dsm_inactive_export_poses",
    "dsm_frame_superpixel_image", "dsm_fuse_stream_window",
    "dsm_publish_enable", "dsm_publish_enqueue", "dsm_publish_wait", "dsm_debug_publish_chunks",
    "dsm_field_enable", "dsm_field_enqueue", "dsm_field_wait",
    "dsm_field_enqueue_resident", "dsm_field_query_enable", "dsm_field_query_enqueue", "dsm_field_query_wait",
    "dsm_views_enable", "dsm_views_capture", "dsm_field_enqueue_known", "dsm_field_state",
    "dsm_frontier_enable", "dsm_frontier_enqueue", "dsm_frontier_wait", "dsm_debug_field_load_state",
    "dsm_field_signed_enable", "dsm_field_signed", "dsm_field_query_enqueue_signed",
    "dsm_reach_enable", "dsm_reach_enqueue", "dsm_reach_enqueue_terrain", "dsm_reach_wait", "dsm_reach_matrix_enable", "dsm_reach_matrix_enqueue",
    "dsm_reach_matrix_enqueue_terrain", "dsm_reach_matrix_wait", "dsm_gain_enable", "dsm_gain_enqueue", "dsm_gain_wait",
    "dsm_tour_enable", "dsm_tour_enqueue", "dsm_tour_wait", "dsm_viewpoint_enable", "dsm_viewpoint_enqueue", "dsm_viewpoint_wait",
    "dsm_viewpoint_enqueue_terrain",
    "dsm_trajectory_enable", "dsm_trajectory_enqueue", "dsm_trajectory_wait",
    "dsm_heading_enable", "dsm_heading_enqueue", "dsm_heading_wait",
    "dsm_terrain_enable", "dsm_terrain_enqueue", "dsm_terrain_wait",
    "dsm_inactive_segments", "dsm_inactive_load", "dsm_map_save", "dsm_map_load", "dsm_map_peek",
    "dsm_checkpoint_enable", "dsm_checkpoint_enqueue", "dsm_checkpoint_wait", "dsm_debug_checkpoint_drain_ctas",
    "dsm_checkpoint_enqueue_incremental", "dsm_map_load_journal", "dsm_map_peek_journal", "dsm_journal_materialize",
    "dsm_checkpoint_views_enable",
    "dsm_comm_unique_id", "dsm_comm_init", "dsm_comm_destroy", "dsm_gather_deltas", "dsm_gather_wait", "dsm_gathered_device",
    "dsm_gathered_rank_bytes", "dsm_gathered_download", "dsm_set_constants", "dsm_set_concurrency",
]


class DsmParams(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32),
                ("fx", ctypes.c_float), ("fy", ctypes.c_float), ("cx", ctypes.c_float), ("cy", ctypes.c_float),
                ("fuse_far", ctypes.c_float), ("fuse_near", ctypes.c_float),
                ("max_batch", ctypes.c_int32), ("max_local_surfels", ctypes.c_int32)]


class DsmConstants(ctypes.Structure):
    _fields_ = [("huber_range", ctypes.c_double), ("baseline", ctypes.c_double), ("disparity_error", ctypes.c_double),
                ("min_tolerate_diff", ctypes.c_double)]


class DsmFieldParams(ctypes.Structure):
    _fields_ = [("voxel", ctypes.c_float), ("nx", ctypes.c_int32), ("ny", ctypes.c_int32), ("nz", ctypes.c_int32)]


# dsm_field_query_wait's result records (include/dsm.h): a point sample and a trajectory clearance
FIELD_SAMPLE_DTYPE = np.dtype([("dist", "<f4"), ("gx", "<f4"), ("gy", "<f4"), ("gz", "<f4")])
CLEARANCE_DTYPE = np.dtype([("min_dist", "<f4"), ("argmin", "<i4"), ("first_hit", "<i4"), ("n_outside", "<i4")])
# dsm_frontier_wait's records (include/dsm.h): a cluster (96 B) and the counts
FRONTIER_CLUSTER_DTYPE = np.dtype([("n_voxels", "<i4"), ("first", "<i4"), ("offset", "<i4"), ("lo", "<i4", 3), ("hi", "<i4", 3),
                                   ("reserved", "<i4"), ("n_faces", "<i8"), ("open", "<i8", 3), ("centroid", "<f8", 3)])
FRONTIER_COUNTS_DTYPE = np.dtype([("n_frontier", "<i4"), ("n_components", "<i4"), ("n_clusters", "<i4"), ("n_listed", "<i4")])
# dsm_reach_wait's records (include/dsm.h): a target (32 B) and the header (64 B)
REACH_TARGET_DTYPE = np.dtype([("cost", "<u4"), ("approach", "<i4"), ("target", "<i4"), ("viewpoint", "<i4"), ("path_offset", "<i4"),
                               ("path_len", "<i4"), ("status", "<i4"), ("reserved", "<i4")])
REACH_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("start_voxel", "<i4"), ("start_status", "<i4"), ("start_approach", "<i4"),
                             ("rounds", "<i4"), ("converged", "<i4"), ("n_traversable", "<i4"), ("n_reached", "<i4"),
                             ("n_goals", "<i4"), ("n_clusters_total", "<i4"), ("n_targets", "<i4"), ("n_path_voxels", "<i4"),
                             ("reserved", "<i4", 2)])
# dsm_reach_matrix_wait's records (include/dsm.h): a site (32 B) and the header (64 B)
REACH_SITE_DTYPE = np.dtype([("voxel", "<i4"), ("status", "<i4"), ("approach", "<i4"), ("rounds", "<i4"), ("converged", "<i4"),
                             ("n_reached", "<i4"), ("reserved", "<i4", 2)])
REACH_MATRIX_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_sites", "<i4"), ("status", "<i4"), ("n_traversable", "<i4"),
                                    ("n_active_tiles", "<i4"), ("max_tiles", "<i4"), ("rounds", "<i4"), ("reserved", "<i4", 7)])
# dsm_gain_wait's records (include/dsm.h): a view's gain (32 B) and the header (32 B)
VIEW_GAIN_DTYPE = np.dtype([("n_frustum", "<i4"), ("n_free", "<i4"), ("n_unknown", "<i4"), ("n_occupied", "<i4"), ("n_frontier", "<i4"),
                            ("n_cluster", "<i4"), ("status", "<i4"), ("reserved", "<i4")])
GAIN_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_views", "<i4"), ("n_clusters_table", "<i4"), ("unknown_blocks", "<i4"),
                            ("reserved", "<i4", 2)])
# dsm_tour_wait's records (include/dsm.h): the header (64 B) and a start (16 B)
TOUR_INFO_DTYPE = np.dtype([("n_sites", "<i4"), ("n_included", "<i4"), ("open", "<i4"), ("n_starts", "<i4"), ("max_passes", "<i4"),
                            ("best_start", "<i4"), ("best_cost", "<i8"), ("seed", "<u8"), ("n_infinite", "<i4"), ("reserved", "<i4", 5)])
TOUR_START_DTYPE = np.dtype([("cost", "<i8"), ("passes", "<i4"), ("converged", "<i4")])
# dsm_viewpoint_wait's records (include/dsm.h): a cluster (32 B), a viewpoint slot (32 B) and the header (64 B)
VIEWPOINT_CLUSTER_DTYPE = np.dtype([("cluster", "<i4"), ("status", "<i4"), ("n_samples", "<i4"), ("n_inside", "<i4"),
                                    ("n_traversable", "<i4"), ("n_reached", "<i4"), ("n_viewpoints", "<i4"), ("reserved", "<i4")])
VIEWPOINT_DTYPE = np.dtype([("voxel", "<i4"), ("offset", "<i4"), ("rotation", "<i4"), ("n_seen", "<i4"), ("cost", "<u4"),
                            ("reserved", "<i4", 3)])
VIEWPOINT_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_clusters", "<i4"), ("n_offsets", "<i4"), ("n_rotations", "<i4"),
                                 ("top_k", "<i4"), ("unknown_blocks", "<i4"), ("with_reach", "<i4"), ("n_clusters_table", "<i4"),
                                 ("reserved", "<i4", 6)])

# dsm_trajectory_wait's records (include/dsm.h): a trajectory (96 B) and the header (64 B)
TRAJECTORY_DTYPE = np.dtype([("status", "<i4"), ("iterations", "<i4"), ("evaluations", "<i4"), ("n_free_outside", "<i4"),
                             ("cost_start", "<f8"), ("cost", "<f8"), ("smoothness", "<f8"), ("clearance", "<f8"),
                             ("feasibility", "<f8"), ("max_v", "<f8"), ("max_a", "<f8"), ("min_dist", "<f4"), ("argmin", "<i4"),
                             ("first_hit", "<i4"), ("n_outside", "<i4"), ("reserved", "<i4", 2)])
TRAJECTORY_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_trajectories", "<i4"), ("n_points", "<i4"), ("n_status", "<i4", 4),
                                  ("reserved", "<i4", 7)])

# dsm_heading_enqueue's per-trajectory request (16 B) and dsm_heading_wait's records (include/dsm.h): a trajectory (32 B),
# a sample (32 B), the counts of one (sample, rotation) (8 B) and the header (64 B)
HEADING_REQUEST_DTYPE = np.dtype([("start", "<i4"), ("end", "<i4"), ("max_step", "<i4"), ("reserved", "<i4")])
HEADING_DTYPE = np.dtype([("status", "<i4"), ("n_samples", "<i4"), ("sample_offset", "<i4"), ("n_outside", "<i4"), ("score", "<i8"),
                          ("steps", "<i4"), ("reserved", "<i4")])
HEADING_SAMPLE_DTYPE = np.dtype([("p", "<f8", 3), ("rotation", "<i4"), ("turn", "<i4")])
HEADING_COUNT_DTYPE = np.dtype([("n_unknown", "<i4"), ("n_frontier", "<i4")])
HEADING_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("n_trajectories", "<i4"), ("n_samples", "<i4"), ("n_rot", "<i4"),
                               ("unknown_blocks", "<i4"), ("n_status", "<i4", 2), ("reserved", "<i4", 7)])

# dsm_terrain_wait's header (include/dsm.h, 64 B)
TERRAIN_INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("m", "<i4", 3), ("up", "<i4"), ("headroom", "<i4"), ("max_step", "<i4"),
                               ("n_support", "<i4"), ("n_blocked", "<i4"), ("n_traversable", "<i4"), ("reserved", "<i4", 4)])


class DsmGainCamera(ctypes.Structure):
    """dsm_gain_camera_t (48 B): pinhole intrinsics, image size, range and the blocking rule of a gain job."""
    _fields_ = [("fx", ctypes.c_double), ("fy", ctypes.c_double), ("cx", ctypes.c_double), ("cy", ctypes.c_double),
                ("width", ctypes.c_int32), ("height", ctypes.c_int32), ("max_range", ctypes.c_float), ("unknown_blocks", ctypes.c_int32)]


class DsmViewpointParams(ctypes.Structure):
    """dsm_viewpoint_params_t (40 B): the candidate ring, sampling, selection and traversability of a viewpoint job."""
    _fields_ = [("r_min", ctypes.c_int32), ("r_max", ctypes.c_int32), ("dz_max", ctypes.c_int32), ("stride", ctypes.c_int32),
                ("max_samples", ctypes.c_int32), ("min_seen", ctypes.c_int32), ("top_k", ctypes.c_int32), ("with_reach", ctypes.c_int32),
                ("radius", ctypes.c_float), ("reserved", ctypes.c_int32)]


class DsmTrajectoryParams(ctypes.Structure):
    """dsm_trajectory_params_t (88 B): the weights, limits and stopping rules of a trajectory job, shared by its
    trajectories."""
    _fields_ = [("w_smooth", ctypes.c_double), ("w_clear", ctypes.c_double), ("w_feas", ctypes.c_double),
                ("margin", ctypes.c_double), ("v_max", ctypes.c_double), ("a_max", ctypes.c_double), ("g_tol", ctypes.c_double),
                ("max_iter", ctypes.c_int32), ("memory", ctypes.c_int32), ("max_ls", ctypes.c_int32), ("samples", ctypes.c_int32),
                ("radius", ctypes.c_float), ("reserved", ctypes.c_int32 * 3)]


CONSTANTS_DRIVE = (0.4, 0.5, 4.0, 0.1)    # fusion_functions.h:13-16
CONSTANTS_RGBD = (0.05, 0.08, 1.0, 0.05)  # fusion_functions.h:18-21


class DsmError(RuntimeError):
    def __init__(self, code, detail=""):
        self.code = code
        super().__init__(f"{ERRORS.get(code, code)}: {detail}")


_lib = None


def load_library():
    """Loads libdsm_b200.so; raises if it has not been built (no fallback of any kind)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(f"{LIB_PATH} not built: run `python -m densesurfelmapping_b200.build` "
                                "(or __graft_entry__.build()); this package has no CPU fallback")
    L = ctypes.CDLL(LIB_PATH)
    vp, ci, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    L.dsm_version.restype = ci
    L.dsm_strerror.restype = ctypes.c_char_p
    L.dsm_strerror.argtypes = [ci]
    L.dsm_last_error.restype = ctypes.c_char_p
    L.dsm_last_error.argtypes = [vp]
    L.dsm_kernel_name.restype = ctypes.c_char_p
    L.dsm_kernel_name.argtypes = [ci]
    L.dsm_create.argtypes = [ctypes.POINTER(DsmParams), ci, vp, ctypes.POINTER(vp)]
    L.dsm_destroy.argtypes = [vp]
    L.dsm_destroy.restype = None
    L.dsm_num_seeds.argtypes = [vp]
    L.dsm_fuse_frame.argtypes = [vp, ci, vp, cs, vp, cs, vp, vp, ci, vp, ci, ctypes.POINTER(ci)]
    L.dsm_batch_upload.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp]
    L.dsm_batch_run.argtypes = [vp]
    L.dsm_batch_download.argtypes = [vp, vp, vp, vp]
    L.dsm_sync.argtypes = [vp]
    L.dsm_fuse_batch.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dsm_fuse_batch_async.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dsm_batch_wait.argtypes = [vp]
    L.dsm_batch_restore_pool.argtypes = [vp]
    L.dsm_pool_upload.argtypes = [vp, vp, ci]
    L.dsm_fuse_frame_resident.argtypes = [vp, ci, vp, cs, vp, cs, vp, ctypes.POINTER(ci)]
    L.dsm_pool_transform.argtypes = [vp, vp]
    L.dsm_fuse_stream_resident.argtypes = [vp, ci, vp, vp, vp, vp, vp]
    L.dsm_fuse_stream_window.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.dsm_publish_enable.argtypes = [vp]
    L.dsm_publish_enqueue.argtypes = [vp, ci]
    L.dsm_publish_wait.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(ci), ctypes.POINTER(vp), ctypes.POINTER(ci), ctypes.POINTER(ci)]
    L.dsm_debug_publish_chunks.argtypes = [vp, ctypes.POINTER(ci)]
    L.dsm_field_enable.argtypes = [vp, ctypes.POINTER(DsmFieldParams)]
    L.dsm_field_enqueue.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ci]
    L.dsm_field_wait.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ci)]
    L.dsm_field_enqueue_resident.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ci]
    L.dsm_field_query_enable.argtypes = [vp, ci, ci, ci]
    L.dsm_field_query_enqueue.argtypes = [vp, vp, ci, vp, vp, ci, ctypes.c_float, ctypes.c_float]
    L.dsm_field_query_wait.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_views_enable.argtypes = [vp, ci, ctypes.c_float]
    L.dsm_views_capture.argtypes = [vp, ci, ci]
    L.dsm_field_enqueue_known.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ci, vp, vp, ci, ci]
    L.dsm_field_state.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(ci)]
    L.dsm_frontier_enable.argtypes = [vp, ci, ci]
    L.dsm_frontier_enqueue.argtypes = [vp, ci]
    L.dsm_frontier_wait.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp), vp]
    L.dsm_debug_field_load_state.argtypes = [vp, vp, ctypes.POINTER(ctypes.c_int32)]
    L.dsm_field_signed_enable.argtypes = [vp]
    L.dsm_field_signed.argtypes = [vp, ctypes.POINTER(vp)]
    L.dsm_field_query_enqueue_signed.argtypes = [vp, vp, ci, vp, vp, ci, ctypes.c_float, ctypes.c_float]
    L.dsm_reach_enable.argtypes = [vp, ci, ci, ci]
    L.dsm_reach_enqueue.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.c_float, ci, vp, ci, ci, ci]
    L.dsm_reach_enqueue_terrain.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.c_float, ci, vp, ci, ci, ci]
    L.dsm_reach_wait.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_reach_matrix_enable.argtypes = [vp, ci, ci, ci]
    L.dsm_reach_matrix_enqueue.argtypes = [vp, vp, ci, ctypes.c_float, ci]
    L.dsm_reach_matrix_enqueue_terrain.argtypes = [vp, vp, ci, ctypes.c_float, ci]
    L.dsm_reach_matrix_wait.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_gain_enable.argtypes = [vp, ci]
    L.dsm_gain_enqueue.argtypes = [vp, ctypes.POINTER(DsmGainCamera), vp, vp, ci]
    L.dsm_gain_wait.argtypes = [vp, vp, ctypes.POINTER(vp)]
    L.dsm_tour_enable.argtypes = [vp, ci, ci]
    L.dsm_tour_enqueue.argtypes = [vp, vp, ci, ci, ci, ci, ctypes.c_uint64]
    L.dsm_tour_wait.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_viewpoint_enable.argtypes = [vp, ci, ci]
    L.dsm_viewpoint_enqueue.argtypes = [vp, ctypes.POINTER(DsmGainCamera), vp, ci, vp, ci, ctypes.POINTER(DsmViewpointParams)]
    L.dsm_viewpoint_enqueue_terrain.argtypes = [vp, ctypes.POINTER(DsmGainCamera), vp, ci, vp, ci, ctypes.POINTER(DsmViewpointParams), ci]
    L.dsm_viewpoint_wait.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_trajectory_enable.argtypes = [vp, ci, ci, ci]
    L.dsm_trajectory_enqueue.argtypes = [vp, vp, vp, vp, ci, ctypes.POINTER(DsmTrajectoryParams)]
    L.dsm_trajectory_wait.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_heading_enable.argtypes = [vp, ci, ci]
    L.dsm_heading_enqueue.argtypes = [vp, vp, vp, ci, ctypes.POINTER(DsmGainCamera), vp, ci, ci, vp, ctypes.c_int32, ctypes.c_int32]
    L.dsm_heading_wait.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_terrain_enable.argtypes = [vp, ci]
    L.dsm_terrain_enqueue.argtypes = [vp, ci, ci]
    L.dsm_terrain_wait.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.dsm_inactive_reserve.argtypes = [vp, ci]
    L.dsm_inactive_retire.argtypes = [vp, ci, ctypes.POINTER(ci)]
    L.dsm_inactive_reactivate.argtypes = [vp, ci, ctypes.POINTER(ci)]
    L.dsm_inactive_transform.argtypes = [vp, ci, vp]
    L.dsm_inactive_export_cloud.argtypes = [vp, vp, ci, ctypes.POINTER(ci)]
    L.dsm_inactive_export_poses.argtypes = [vp, vp, ci, vp, ci, ctypes.POINTER(ci)]
    L.dsm_frame_superpixel_image.argtypes = [vp, ci, vp, ctypes.c_size_t]
    L.dsm_frame_raw_cloud.argtypes = [vp, ci, vp, vp, ci, ctypes.POINTER(ci)]
    L.dsm_inactive_download.argtypes = [vp, ci, vp, ci, ctypes.POINTER(ci)]
    L.dsm_inactive_size.argtypes = [vp, ctypes.POINTER(ci), ctypes.POINTER(ci)]
    L.dsm_inactive_segments.argtypes = [vp, vp, ci, ctypes.POINTER(ci)]
    L.dsm_inactive_load.argtypes = [vp, vp, ci, vp, ci]
    L.dsm_map_save.argtypes = [vp, ctypes.c_char_p, vp, cs]
    L.dsm_map_load.argtypes = [vp, ctypes.c_char_p, vp, cs, ctypes.POINTER(cs)]
    L.dsm_map_peek.argtypes = [ctypes.c_char_p, vp, cs, ctypes.POINTER(cs), vp, ci, ctypes.POINTER(ci)]
    L.dsm_checkpoint_enable.argtypes = [vp]
    L.dsm_checkpoint_views_enable.argtypes = [vp]
    L.dsm_checkpoint_enqueue.argtypes = [vp, ctypes.c_char_p, vp, cs]
    L.dsm_checkpoint_wait.argtypes = [vp, ci, ctypes.POINTER(ci)]
    L.dsm_debug_checkpoint_drain_ctas.argtypes = [vp, ci]
    L.dsm_checkpoint_enqueue_incremental.argtypes = [vp, ctypes.c_char_p, vp, cs]
    L.dsm_map_load_journal.argtypes = [vp, ctypes.c_char_p, vp, cs, ctypes.POINTER(cs), ctypes.POINTER(ci)]
    L.dsm_map_peek_journal.argtypes = [ctypes.c_char_p, vp, cs, ctypes.POINTER(cs), vp, ci, ctypes.POINTER(ci), ctypes.POINTER(ci)]
    L.dsm_journal_materialize.argtypes = [ctypes.c_char_p, ctypes.c_char_p]
    L.dsm_pool_retire.argtypes = [vp, ci, vp, ci, ctypes.POINTER(ci)]
    L.dsm_pool_append.argtypes = [vp, vp, ci]
    L.dsm_pool_size.argtypes = [vp, ctypes.POINTER(ci)]
    L.dsm_pool_download.argtypes = [vp, vp, ci, ctypes.POINTER(ci)]
    L.dsm_get_labels.argtypes = [vp, ci, vp]
    L.dsm_get_seeds.argtypes = [vp, ci, vp]
    L.dsm_debug_stop_after.argtypes = [vp, ci]
    L.dsm_debug_invariant_violations.argtypes = [vp, ctypes.POINTER(ci)]
    L.dsm_profile_enable.argtypes = [vp, ctypes.c_uint32]
    L.dsm_profile_reset.argtypes = [vp]
    L.dsm_profile_read.argtypes = [vp, vp, vp]
    L.dsm_device_buffer.argtypes = [vp, ci, ctypes.POINTER(vp), ctypes.POINTER(cs)]
    L.dsm_pool_export_cloud.argtypes = [vp, ci, vp, ci, ctypes.POINTER(ci)]
    L.dsm_pool_export_surfels.argtypes = [vp, ci, vp, ci, ctypes.POINTER(ci)]
    L.dsm_write_pcd.argtypes = [ctypes.c_char_p, vp, cs, ci]
    L.dsm_write_ply_mesh.argtypes = [ctypes.c_char_p, vp, cs]
    L.dsm_mesh_vertices.argtypes = [vp, cs, vp]
    L.dsm_set_constants.argtypes = [vp, ctypes.POINTER(DsmConstants)]
    L.dsm_set_concurrency.argtypes = [vp, ctypes.c_int]
    L.dsm_comm_unique_id.argtypes = [vp]
    L.dsm_comm_init.argtypes = [vp, vp, ci, ci]
    L.dsm_comm_destroy.argtypes = [vp]
    L.dsm_gather_deltas.argtypes = [vp, ci]
    L.dsm_gather_wait.argtypes = [vp]
    L.dsm_gathered_device.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(cs)]
    L.dsm_gathered_rank_bytes.argtypes = [vp, ci, ctypes.POINTER(cs)]
    L.dsm_gathered_download.argtypes = [vp, ci, vp, cs]
    _lib = L
    return L


def comm_unique_id() -> bytes:
    """128-byte NCCL unique id (rank 0 creates it and hands it to the other ranks out of band)."""
    L = load_library()
    buf = ctypes.create_string_buffer(128)
    rc = L.dsm_comm_unique_id(buf)
    if rc != DSM_OK:
        raise DsmError(rc, L.dsm_strerror(rc).decode())
    return buf.raw


def kernel_names():
    L = load_library()
    return [L.dsm_kernel_name(i).decode() for i in range(NUM_KERNELS)]


def _ptr(a):
    return None if a is None else a.ctypes.data


def _take(ptr, n, dtype):
    """A numpy copy of n records of dtype at the address in ptr (a c_void_p); empty for n == 0 or a null pointer."""
    dtype = np.dtype(dtype)
    if n == 0 or not ptr.value:
        return np.zeros(0, dtype)
    return np.frombuffer((ctypes.c_uint8 * (n * dtype.itemsize)).from_address(ptr.value), dtype=dtype).copy()


def _camera(camera):
    """The DsmGainCamera of (fx, fy, cx, cy, width, height, max_range, unknown_blocks)."""
    return DsmGainCamera(*[float(x) for x in camera[:4]], int(camera[4]), int(camera[5]), float(camera[6]), int(camera[7]))


def window_lists(per_frame):
    """One list of keyframes per frame -> (keys, offsets[n + 1]) as dsm_fuse_stream_window takes them."""
    lens = [len(x) for x in per_frame]
    ofs = np.zeros(len(lens) + 1, dtype=np.int32)
    ofs[1:] = np.cumsum(lens)
    keys = np.concatenate([np.asarray(x, dtype=np.int32).reshape(-1) for x in per_frame] + [np.zeros(1, np.int32)])
    return np.ascontiguousarray(keys, dtype=np.int32), ofs


def pose16(pose):
    """Eigen::Matrix4f memory order (column-major float32[16]) of a pose.  A flat 16-vector is taken as already
    column-major (what synth.pose_stream returns); a (4, 4) array is taken as the MATRIX T_world<-cam the way numpy
    writes it (row i, column j = pose[i, j]) and is transposed into column-major memory -- it is not reinterpreted."""
    a = np.asarray(pose, dtype=np.float32)
    if a.shape == (4, 4):
        return np.ascontiguousarray(a.T).reshape(16)
    if a.size != 16:
        raise ValueError("pose must be a (4, 4) matrix or a column-major 16-vector")
    return np.ascontiguousarray(a).reshape(16)


class Context:
    """Owns one dsm_ctx (one per GPU)."""

    def __init__(self, cam, max_batch=1, max_local_surfels=1 << 20, device=0, cuda_stream=None):
        self.lib = load_library()
        self.cam = cam
        self.S = num_seeds(cam.width, cam.height)
        self.max_batch = max_batch
        p = DsmParams(cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, cam.far, cam.near,
                      max_batch, max_local_surfels)
        h = ctypes.c_void_p()
        rc = self.lib.dsm_create(ctypes.byref(p), device, cuda_stream, ctypes.byref(h))
        if rc != DSM_OK:
            raise DsmError(rc, self.lib.dsm_strerror(rc).decode())
        self.h = h

    def _ck(self, rc):
        if rc != DSM_OK:
            raise DsmError(rc, self.lib.dsm_last_error(self.h).decode() or self.lib.dsm_strerror(rc).decode())

    def _waited(self, rc, name, results):
        """The results of a wait that returned rc: results() builds them once rc is DSM_OK or DSM_E_CAPACITY (any other
        code raises first); DSM_E_CAPACITY raises DsmError carrying them as attribute `name`."""
        if rc not in (DSM_OK, DSM_E_CAPACITY):
            self._ck(rc)
        out = results()
        if rc != DSM_OK:
            err = DsmError(rc, self.lib.dsm_last_error(self.h).decode())
            setattr(err, name, out)
            raise err
        return out

    def close(self):
        if getattr(self, "h", None):
            self.lib.dsm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- reference-identical single frame ----
    def fuse_frame(self, ref_idx, gray, depth, pose, local):
        gray = np.ascontiguousarray(gray, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        pose = pose16(pose)
        local = np.array(local, dtype=SURFEL_DTYPE, copy=True)
        new = np.zeros(self.S, dtype=SURFEL_DTYPE)
        n = ctypes.c_int(0)
        self._ck(self.lib.dsm_fuse_frame(self.h, int(ref_idx), _ptr(gray), gray.strides[0], _ptr(depth), depth.strides[0],
                                         _ptr(pose), _ptr(local) if len(local) else None, len(local),
                                         _ptr(new), self.S, ctypes.byref(n)))
        return local, new[:n.value].copy()

    # ---- batch stages ----
    def batch_upload(self, ref_idx, gray, depth, poses, local, offsets):
        self._keep = (np.ascontiguousarray(ref_idx, dtype=np.int32), np.ascontiguousarray(gray, dtype=np.uint8),
                      np.ascontiguousarray(depth, dtype=np.float32), np.ascontiguousarray(poses, dtype=np.float32),
                      np.ascontiguousarray(local, dtype=SURFEL_DTYPE), np.ascontiguousarray(offsets, dtype=np.int32))
        r, g, d, p, l, o = self._keep
        n = len(r)
        assert g.shape == (n, self.cam.height, self.cam.width) and d.shape == g.shape and len(o) == n + 1
        self.nb = n
        self.n_pool = int(o[-1])
        self._ck(self.lib.dsm_batch_upload(self.h, n, _ptr(r), _ptr(g), _ptr(d), _ptr(p), _ptr(l) if len(l) else None, _ptr(o)))

    def batch_run(self):
        self._ck(self.lib.dsm_batch_run(self.h))

    def batch_restore_pool(self):
        self._ck(self.lib.dsm_batch_restore_pool(self.h))

    def sync(self):
        self._ck(self.lib.dsm_sync(self.h))

    def batch_download(self):
        local = np.zeros(self.n_pool, dtype=SURFEL_DTYPE)
        new = np.zeros((self.nb, self.S), dtype=SURFEL_DTYPE)
        cnt = np.zeros(self.nb, dtype=np.int32)
        self._ck(self.lib.dsm_batch_download(self.h, _ptr(local) if self.n_pool else None, _ptr(new), _ptr(cnt)))
        self.sync()
        return local, [new[b, :cnt[b]].copy() for b in range(self.nb)]

    def fuse_batch(self, ref_idx, gray, depth, poses, local, offsets):
        self.batch_upload(ref_idx, gray, depth, poses, local, offsets)
        self.batch_run()
        return self.batch_download()

    def set_constants(self, constants):
        """(huber_range, baseline, disparity_error, min_tolerate_diff): CONSTANTS_DRIVE (default) or CONSTANTS_RGBD."""
        k = DsmConstants(*constants)
        self._ck(self.lib.dsm_set_constants(self.h, ctypes.byref(k)))

    def set_concurrency(self, sub_batches: int):
        """Concurrent sub-batches of batch_run (1..4, default 2); 1 for clean per-kernel profile durations."""
        self._ck(self.lib.dsm_set_concurrency(self.h, int(sub_batches)))

    # ---- multi-GPU gather of the surfel deltas (csrc/dsm_comm.cu) ----
    def comm_init(self, unique_id: bytes, rank: int, nranks: int):
        assert len(unique_id) == 128
        buf = ctypes.create_string_buffer(bytes(unique_id), 128)
        self._ck(self.lib.dsm_comm_init(self.h, buf, int(rank), int(nranks)))
        self.comm_rank, self.comm_size = rank, nranks

    def gather_deltas(self, root=0):
        self._ck(self.lib.dsm_gather_deltas(self.h, int(root)))

    def gather_wait(self):
        self._ck(self.lib.dsm_gather_wait(self.h))

    def gathered_payload(self, rank):
        """root only: the payload rank `rank` sent in the last gather, as a uint8 array (see gather.unpack_payload)."""
        n = ctypes.c_size_t(0)
        self._ck(self.lib.dsm_gathered_rank_bytes(self.h, int(rank), ctypes.byref(n)))
        out = np.zeros(n.value, np.uint8)
        self._ck(self.lib.dsm_gathered_download(self.h, int(rank), _ptr(out), n.value))
        return out

    # ---- GPU-resident pool (stream mode) ----
    def pool_upload(self, local):
        local = np.ascontiguousarray(local, dtype=SURFEL_DTYPE)
        self._ck(self.lib.dsm_pool_upload(self.h, _ptr(local) if len(local) else None, len(local)))

    def fuse_frame_resident(self, ref_idx, gray, depth, pose, want_count=False):
        gray = np.ascontiguousarray(gray, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        pose = pose16(pose)
        n = ctypes.c_int(0)
        self._ck(self.lib.dsm_fuse_frame_resident(self.h, int(ref_idx), _ptr(gray), gray.strides[0], _ptr(depth), depth.strides[0],
                                                  _ptr(pose), ctypes.byref(n) if want_count else None))
        return n.value if want_count else None

    def fuse_stream_resident(self, ref_idx, gray, depth, poses, want_counts=False):
        """n consecutive frames of one stream in one call (see include/dsm.h); gray [n,H,W] u8, depth [n,H,W] f32."""
        ref = np.ascontiguousarray(ref_idx, dtype=np.int32)
        gray = np.ascontiguousarray(gray, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        poses = np.ascontiguousarray(poses, dtype=np.float32).reshape(len(ref), 16)
        assert gray.shape == (len(ref), self.cam.height, self.cam.width) and depth.shape == gray.shape
        cnt = np.zeros(len(ref), dtype=np.int32)
        self._ck(self.lib.dsm_fuse_stream_resident(self.h, len(ref), _ptr(ref), _ptr(gray), _ptr(depth), _ptr(poses),
                                                   _ptr(cnt) if want_counts else None))
        return cnt if want_counts else None

    def fuse_stream_window(self, ref_idx, gray, depth, poses, retire, reactivate, want_counts=False):
        """fuse_stream_resident with each frame's move_add_surfels in front of its fuse (see include/dsm.h).
        retire / reactivate: one list of keyframe indices per frame (poses_to_remove / poses_to_add of the node).
        want_counts: synchronise and return the new surfels per frame (-1: frame not applied); a rejected frame then
        raises DsmError(DSM_E_CAPACITY) with the counts in .counts."""
        ref = np.ascontiguousarray(ref_idx, dtype=np.int32)
        n = len(ref)
        gray = np.ascontiguousarray(gray, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        poses = np.ascontiguousarray(poses, dtype=np.float32).reshape(n, 16)
        assert gray.shape == (n, self.cam.height, self.cam.width) and depth.shape == gray.shape
        assert len(retire) == n and len(reactivate) == n
        rk, ro = window_lists(retire)
        ak, ao = window_lists(reactivate)
        cnt = np.zeros(n, dtype=np.int32)
        rc = self.lib.dsm_fuse_stream_window(self.h, n, _ptr(ref), _ptr(gray), _ptr(depth), _ptr(poses), _ptr(rk), _ptr(ro),
                                             _ptr(ak), _ptr(ao), _ptr(cnt) if want_counts else None)
        if rc != DSM_OK:
            err = DsmError(rc, self.lib.dsm_last_error(self.h).decode() or self.lib.dsm_strerror(rc).decode())
            err.counts = cnt if want_counts else None
            raise err
        return cnt if want_counts else None

    def pool_transform(self, W_colmajor):
        w = pose16(W_colmajor)
        self._ck(self.lib.dsm_pool_transform(self.h, _ptr(w)))

    def _read(self, fn, dtype, cap, *args):
        """fn(h, *args, out, cap, &n): the first min(n, cap) records the library wrote."""
        out = np.zeros(max(cap, 1), dtype=dtype)
        n = ctypes.c_int(0)
        self._ck(fn(self.h, *args, _ptr(out), cap, ctypes.byref(n)))
        return out[:min(n.value, cap)].copy()

    def pool_retire(self, keyframe_index, cap=None):
        cap = self.pool_size() if cap is None else cap
        return self._read(self.lib.dsm_pool_retire, SURFEL_DTYPE, cap, int(keyframe_index))

    def pool_append(self, surfels):
        surfels = np.ascontiguousarray(surfels, dtype=SURFEL_DTYPE)
        self._ck(self.lib.dsm_pool_append(self.h, _ptr(surfels) if len(surfels) else None, len(surfels)))

    def pool_size(self):
        n = ctypes.c_int(0)
        self._ck(self.lib.dsm_pool_size(self.h, ctypes.byref(n)))
        return n.value

    def pool_download(self):
        n = self.pool_size()
        out = np.zeros(n, dtype=SURFEL_DTYPE)
        c = ctypes.c_int(0)
        self._ck(self.lib.dsm_pool_download(self.h, _ptr(out) if n else None, n, ctypes.byref(c)))
        return out[:c.value]

    def pool_export_cloud(self, min_update_times=5, cap=None):
        """publish_active_pointcloud & co. (surfel_map.cpp:1398-1417): POINT_DTYPE array in pool order."""
        cap = self.pool_size() if cap is None else cap
        return self._read(self.lib.dsm_pool_export_cloud, POINT_DTYPE, cap, int(min_update_times))

    def pool_export_surfels(self, min_update_times=5, cap=None):
        cap = self.pool_size() if cap is None else cap
        return self._read(self.lib.dsm_pool_export_surfels, SURFEL_DTYPE, cap, int(min_update_times))

    # ---- inactive store ----
    def inactive_reserve(self, n):
        self._ck(self.lib.dsm_inactive_reserve(self.h, int(n)))

    def inactive_retire(self, keyframe_index):
        n = ctypes.c_int(0)
        self._ck(self.lib.dsm_inactive_retire(self.h, int(keyframe_index), ctypes.byref(n)))
        return n.value

    def inactive_reactivate(self, keyframe_index):
        n = ctypes.c_int(0)
        self._ck(self.lib.dsm_inactive_reactivate(self.h, int(keyframe_index), ctypes.byref(n)))
        return n.value

    def inactive_transform(self, keyframe_index, W_colmajor):
        w = pose16(W_colmajor)
        self._ck(self.lib.dsm_inactive_transform(self.h, int(keyframe_index), _ptr(w)))

    def inactive_size(self):
        a, b = ctypes.c_int(0), ctypes.c_int(0)
        self._ck(self.lib.dsm_inactive_size(self.h, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def inactive_download(self, keyframe_index=-1):
        return self._read(self.lib.dsm_inactive_download, SURFEL_DTYPE, self.inactive_size()[0], int(keyframe_index))

    def inactive_export_cloud(self):
        return self._read(self.lib.dsm_inactive_export_cloud, POINT_DTYPE, self.inactive_size()[0])

    def inactive_export_poses(self, keyframes, cap=None):
        """The inactive half of publish_neighbor_pointcloud (surfel_map.cpp:1306-1321): the stored points of each listed
        keyframe, list order; keyframes with nothing stored contribute nothing.  POINT_DTYPE array."""
        kf = np.ascontiguousarray(keyframes, dtype=np.int32).reshape(-1)
        cap = self.inactive_size()[0] if cap is None else cap
        return self._read(self.lib.dsm_inactive_export_poses, POINT_DTYPE, cap, _ptr(kf) if len(kf) else None, len(kf))

    # ---- checkpoint and resume (DESIGN.md §8.4) ----
    def inactive_segments(self):
        """The store's segment table in store order: int32 [n, 3] of (keyframe, offset, count)."""
        return self._read(self.lib.dsm_inactive_segments, np.dtype((np.int32, 3)), self.inactive_size()[1])

    def inactive_load(self, surfels, segments):
        """Replaces the store's contents (SURFEL_DTYPE, store order) and its table ([n, 3] of (keyframe, offset, count))."""
        surfels = np.ascontiguousarray(surfels, dtype=SURFEL_DTYPE)
        seg = np.ascontiguousarray(segments, dtype=np.int32).reshape(-1, 3)
        self._ck(self.lib.dsm_inactive_load(self.h, _ptr(surfels) if len(surfels) else None, len(surfels),
                                            _ptr(seg) if len(seg) else None, len(seg)))

    def map_save(self, path, extra=b""):
        """The pool, the store, its table and the caller's `extra` bytes to one checkpoint file."""
        buf = ctypes.create_string_buffer(bytes(extra), max(len(extra), 1))
        self._ck(self.lib.dsm_map_save(self.h, os.fsencode(path), buf if len(extra) else None, len(extra)))

    def map_load(self, path) -> bytes:
        """Replaces the map by a checkpoint's and returns its extra bytes."""
        size = ctypes.c_size_t(0)
        rc = self.lib.dsm_map_load(self.h, os.fsencode(path), None, 0, ctypes.byref(size))
        if rc == -6 and size.value > 0:  # the size-then-read of the extra section: nothing was loaded yet
            buf = ctypes.create_string_buffer(size.value)
            self._ck(self.lib.dsm_map_load(self.h, os.fsencode(path), buf, size.value, ctypes.byref(size)))
            return buf.raw[:size.value]
        self._ck(rc)
        return b""

    # ---- checkpoints that do not stop the stream (DESIGN.md §8.5) ----
    def checkpoint_enable(self):
        self._ck(self.lib.dsm_checkpoint_enable(self.h))

    def checkpoint_enqueue(self, path, extra=b""):
        """Enqueues the file map_save(path, extra) would write at this position in the stream; written by the context's
        thread while the caller goes on."""
        buf = ctypes.create_string_buffer(bytes(extra), max(len(extra), 1))
        self._ck(self.lib.dsm_checkpoint_enqueue(self.h, os.fsencode(path), buf if len(extra) else None, len(extra)))

    def checkpoint_wait(self, block=True):
        """True once the enqueued checkpoint's file is written (and the checkpoint retired), False while the write runs
        (block=False only).  A failed write raises DsmError and retires the checkpoint."""
        fin = ctypes.c_int(0)
        self._ck(self.lib.dsm_checkpoint_wait(self.h, 1 if block else 0, ctypes.byref(fin)))
        return bool(fin.value)

    # ---- incremental checkpoints (DESIGN.md §8.6) ----
    def checkpoint_enqueue_incremental(self, path, extra=b""):
        """checkpoint_enqueue, but written as one journal record of the changed chunks beside the base at `path`, or as a
        new base; checkpoint_wait retires it."""
        buf = ctypes.create_string_buffer(bytes(extra), max(len(extra), 1))
        self._ck(self.lib.dsm_checkpoint_enqueue_incremental(self.h, os.fsencode(path), buf if len(extra) else None, len(extra)))

    def checkpoint_views_enable(self):
        """Every checkpoint from now on carries the captured views, and every load replaces them (DESIGN.md §8.18)."""
        self._ck(self.lib.dsm_checkpoint_views_enable(self.h))

    def map_load_journal(self, path):
        """map_load of the state base + journal resolve to: (extra bytes, records applied)."""
        size, rec = ctypes.c_size_t(0), ctypes.c_int(0)
        rc = self.lib.dsm_map_load_journal(self.h, os.fsencode(path), None, 0, ctypes.byref(size), ctypes.byref(rec))
        if rc == -6 and size.value > 0:  # the size-then-read of the extra section: nothing was loaded yet
            buf = ctypes.create_string_buffer(size.value)
            self._ck(self.lib.dsm_map_load_journal(self.h, os.fsencode(path), buf, size.value, ctypes.byref(size), ctypes.byref(rec)))
            return buf.raw[:size.value], rec.value
        self._ck(rc)
        return b"", rec.value

    # ---- publishing from inside the stream ----
    def publish_enable(self):
        self._ck(self.lib.dsm_publish_enable(self.h))

    def publish_enqueue(self, min_update_times=5):
        self._ck(self.lib.dsm_publish_enqueue(self.h, int(min_update_times)))

    def publish_wait(self):
        """(active, inactive, inactive_changed_from) of the enqueued snapshot: POINT_DTYPE copies of the context's pinned
        buffers.  A snapshot taken after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as
        `.clouds` (the map of the last applied frame)."""
        pa, pi = ctypes.c_void_p(), ctypes.c_void_p()
        na, ni, cf = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
        rc = self.lib.dsm_publish_wait(self.h, ctypes.byref(pa), ctypes.byref(na), ctypes.byref(pi), ctypes.byref(ni), ctypes.byref(cf))
        return self._waited(rc, "clouds", lambda: (_take(pa, na.value, POINT_DTYPE), _take(pi, ni.value, POINT_DTYPE), cf.value))

    def publish_chunks(self):
        """256-point chunks of the inactive cloud the last waited snapshot forwarded to the host."""
        n = ctypes.c_int(0)
        self._ck(self.lib.dsm_debug_publish_chunks(self.h, ctypes.byref(n)))
        return n.value

    # ---- the map as a distance field ----
    def field_enable(self, voxel, nx, ny, nz):
        p = DsmFieldParams(float(voxel), int(nx), int(ny), int(nz))
        self._ck(self.lib.dsm_field_enable(self.h, ctypes.byref(p)))
        self._field_shape = (int(nz), int(ny), int(nx))

    def field_enqueue(self, center, min_update_times=5, host_copy=True):
        """host_copy=False: dsm_field_enqueue_resident, the grid stays on the device for field_query_*."""
        c = (ctypes.c_double * 3)(*[float(v) for v in center])
        fn = self.lib.dsm_field_enqueue if host_copy else self.lib.dsm_field_enqueue_resident
        self._ck(fn(self.h, c, int(min_update_times)))

    def field_wait(self):
        """(dist, origin, n_occupied) of the enqueued field: dist a float32 [nz][ny][nx] copy of the context's pinned
        buffer (None for a resident field), origin an int32 (3,) array (x, y, z).  A field requested after a rejected
        frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.field` (the map of the last applied frame)."""
        ptr, org, nocc = ctypes.c_void_p(), (ctypes.c_int32 * 3)(), ctypes.c_int(0)
        rc = self.lib.dsm_field_wait(self.h, ctypes.byref(ptr), org, ctypes.byref(nocc))

        def field():
            shape = self._field_shape
            dist = _take(ptr, shape[0] * shape[1] * shape[2], np.float32).reshape(shape) if ptr.value else None
            return dist, np.array(org[:], dtype=np.int32), nocc.value
        return self._waited(rc, "field", field)

    # ---- the signed distance field ----
    def field_signed_enable(self):
        """Every field request from now on also builds the signed grid (negative depth inside the sites)."""
        self._ck(self.lib.dsm_field_signed_enable(self.h))

    def field_signed(self):
        """The signed grid of the last waited field: a float32 [nz][ny][nx] copy of the context's pinned buffer, or None
        for a resident field.  A field requested after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the
        same value as `.signed` (the grid of the last applied frame)."""
        ptr = ctypes.c_void_p()
        rc = self.lib.dsm_field_signed(self.h, ctypes.byref(ptr))

        def grid():
            shape = self._field_shape
            return _take(ptr, shape[0] * shape[1] * shape[2], np.float32).reshape(shape) if ptr.value else None
        return self._waited(rc, "signed", grid)

    # ---- free versus unknown space ----
    def views_enable(self, max_views, max_range):
        self._ck(self.lib.dsm_views_enable(self.h, int(max_views), float(max_range)))

    def views_capture(self, frame, slot):
        """The rays of frame `frame` of the most recent call that took images into slot `slot` (asynchronous)."""
        self._ck(self.lib.dsm_views_capture(self.h, int(frame), int(slot)))

    def field_enqueue_known(self, center, min_update_times, slots, poses, host_copy=True):
        """A known-space field over the captured slots at poses (n, 12) or (n, 3, 4) fp64 [R | t], camera to world;
        field_wait then returns its distances and field_state its voxel states."""
        c = (ctypes.c_double * 3)(*[float(v) for v in center])
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        ps = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
        n = len(sl)
        if ps.shape[0] != n:   # the library reads n poses
            raise ValueError(f"{n} slots and {ps.shape[0]} poses")
        self._ck(self.lib.dsm_field_enqueue_known(self.h, c, int(min_update_times), sl.ctypes.data if n else None,
                                                  ps.ctypes.data if n else None, n, 1 if host_copy else 0))

    def field_state(self):
        """(state, n_free) of the last waited known field: state a uint8 [nz][ny][nx] copy (0 unknown, 1 occupied,
        2 free; None for a field kept on the device)."""
        ptr, nfree = ctypes.c_void_p(), ctypes.c_int(0)
        self._ck(self.lib.dsm_field_state(self.h, ctypes.byref(ptr), ctypes.byref(nfree)))
        state = None
        if ptr.value:
            shape = self._field_shape
            buf = (ctypes.c_uint8 * (shape[0] * shape[1] * shape[2])).from_address(ptr.value)
            state = np.frombuffer(buf, dtype=np.uint8).reshape(shape).copy()
        return state, nfree.value

    def debug_field_load_state(self, state, origin):
        """Makes the uint8 state grid [nz][ny][nx] at integer origin (x, y, z) the latest known field request; field_wait
        and field_state then read it like any other."""
        st = np.ascontiguousarray(state, np.uint8)
        if st.shape != self._field_shape:   # the library reads nx * ny * nz bytes
            raise ValueError(f"state grid {st.shape}, field {self._field_shape}")
        org = (ctypes.c_int32 * 3)(*[int(v) for v in origin])
        self._ck(self.lib.dsm_debug_field_load_state(self.h, st.ctypes.data, org))

    # ---- exploration frontiers of the latest known field ----
    def frontier_enable(self, max_clusters, max_voxels):
        self._ck(self.lib.dsm_frontier_enable(self.h, int(max_clusters), int(max_voxels)))
        self._frontier_caps = (int(max_clusters), int(max_voxels))

    def frontier_enqueue(self, min_voxels=1):
        self._ck(self.lib.dsm_frontier_enqueue(self.h, int(min_voxels)))

    def frontier_wait(self):
        """(clusters, voxels, counts): numpy copies of the context's pinned results, FRONTIER_CLUSTER_DTYPE
        (min(n_clusters, max_clusters),), int32 (n_listed,) and a FRONTIER_COUNTS_DTYPE record.  A job on a field taken
        after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.frontier`."""
        pc, pv = ctypes.c_void_p(), ctypes.c_void_p()
        counts = np.zeros(1, FRONTIER_COUNTS_DTYPE)
        rc = self.lib.dsm_frontier_wait(self.h, ctypes.byref(pc), ctypes.byref(pv), counts.ctypes.data)
        c = counts[0]

        def frontier():
            n_tab = min(int(c["n_clusters"]), self._frontier_caps[0])
            return _take(pc, n_tab, FRONTIER_CLUSTER_DTYPE), _take(pv, int(c["n_listed"]), np.int32), c
        return self._waited(rc, "frontier", frontier)

    # ---- paths through known free space of the latest known field ----
    def reach_enable(self, max_targets, max_path_voxels, max_rounds):
        self._ck(self.lib.dsm_reach_enable(self.h, int(max_targets), int(max_path_voxels), int(max_rounds)))

    def reach_enqueue(self, start, radius, approach, goals=None, with_frontiers=False, host_copy=False):
        """start: a world point (x, y, z); goals: world points, an (n, 3) array-like of float64 (None for none)."""
        self._reach_enqueue(self.lib.dsm_reach_enqueue, False, start, radius, approach, goals, with_frontiers, host_copy)

    def reach_enqueue_terrain(self, start, radius, approach, goals=None, with_frontiers=False, host_copy=False):
        """The reach job on the plane of the latest terrain job (DESIGN.md §8.21), arguments as reach_enqueue's; each
        point stands for its column.  reach_wait then returns the cost grid [m2][m1][m0] of the terrain grid."""
        self._reach_enqueue(self.lib.dsm_reach_enqueue_terrain, True, start, radius, approach, goals, with_frontiers, host_copy)

    def _reach_enqueue(self, call, terrain, start, radius, approach, goals, with_frontiers, host_copy):
        st = (ctypes.c_double * 3)(*[float(v) for v in start])
        g = np.ascontiguousarray(np.zeros((0, 3)) if goals is None else goals, np.float64).reshape(-1, 3)
        self._ck(call(self.h, st, float(radius), int(approach), g.ctypes.data if len(g) else None, len(g), int(bool(with_frontiers)),
                      int(bool(host_copy))))
        self._reach_terrain = terrain   # which grid reach_wait's cost grid covers

    def reach_wait(self):
        """(info, targets, path, cost): numpy copies of the context's pinned results, a REACH_INFO_DTYPE record,
        REACH_TARGET_DTYPE (n_targets,), int32 (n_path_voxels,) and the uint32 cost grid (None without host_copy),
        [nz][ny][nx] after reach_enqueue and [m2][m1][m0] of the terrain grid after reach_enqueue_terrain.  A job on a
        field taken after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.reach`."""
        pt, pp, pc = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        info = np.zeros(1, REACH_INFO_DTYPE)
        rc = self.lib.dsm_reach_wait(self.h, info.ctypes.data, ctypes.byref(pt), ctypes.byref(pp), ctypes.byref(pc))
        i = info[0]

        def reach():
            shape = self._field_shape
            if getattr(self, "_reach_terrain", False):   # the field grid collapsed along the terrain's up axis
                shape = tuple(1 if k == 2 - (abs(self._terrain_up) - 1) else n for k, n in enumerate(shape))
            cost = _take(pc, shape[0] * shape[1] * shape[2], np.uint32).reshape(shape) if pc.value else None
            return i, _take(pt, int(i["n_targets"]), REACH_TARGET_DTYPE), _take(pp, int(i["n_path_voxels"]), np.int32), cost
        return self._waited(rc, "reach", reach)

    # ---- travel costs between many sites through the known free space of the latest known field ----
    def reach_matrix_enable(self, max_sites, max_tiles, max_rounds):
        self._ck(self.lib.dsm_reach_matrix_enable(self.h, int(max_sites), int(max_tiles), int(max_rounds)))

    def reach_matrix_enqueue(self, points, radius, approach):
        """points: world points, an (n, 3) array-like of float64, n >= 1."""
        self._reach_matrix_enqueue(self.lib.dsm_reach_matrix_enqueue, points, radius, approach)

    def reach_matrix_enqueue_terrain(self, points, radius, approach):
        """The matrix job on the plane of the latest terrain job (DESIGN.md §8.22), arguments as reach_matrix_enqueue's;
        each point stands for its column, and the site voxels reach_matrix_wait returns are cells q P + p of that plane."""
        self._reach_matrix_enqueue(self.lib.dsm_reach_matrix_enqueue_terrain, points, radius, approach)

    def _reach_matrix_enqueue(self, call, points, radius, approach):
        p = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
        self._ck(call(self.h, p.ctypes.data if len(p) else None, len(p), float(radius), int(approach)))

    def reach_matrix_wait(self):
        """(info, sites, matrix): numpy copies of the context's pinned results, a REACH_MATRIX_INFO_DTYPE record,
        REACH_SITE_DTYPE (n_sites,) and the uint32 matrix (n_sites, n_sites), row i from site i.  A job on a field taken
        after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.reach_matrix`."""
        ps, pm = ctypes.c_void_p(), ctypes.c_void_p()
        info = np.zeros(1, REACH_MATRIX_INFO_DTYPE)
        rc = self.lib.dsm_reach_matrix_wait(self.h, info.ctypes.data, ctypes.byref(ps), ctypes.byref(pm))
        i = info[0]
        n = int(i["n_sites"])
        return self._waited(rc, "reach_matrix", lambda: (i, _take(ps, n, REACH_SITE_DTYPE), _take(pm, n * n, np.uint32).reshape(n, n)))

    # ---- view gain against the latest known field ----
    def gain_enable(self, max_views):
        self._ck(self.lib.dsm_gain_enable(self.h, int(max_views)))

    def gain_enqueue(self, camera, poses, clusters=None):
        """camera: (fx, fy, cx, cy, width, height, max_range, unknown_blocks); poses: (n, 12) row-major [R | t], camera to
        world; clusters: n frontier-table indices (-1: none), or None when no view names a cluster."""
        cam = _camera(camera)
        P = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
        c = None if clusters is None else np.ascontiguousarray(clusters, np.int32).reshape(-1)
        if c is not None and len(c) != len(P):
            raise ValueError(f"{len(c)} clusters for {len(P)} views")
        self._ck(self.lib.dsm_gain_enqueue(self.h, ctypes.byref(cam), P.ctypes.data if len(P) else None,
                                           None if c is None else c.ctypes.data, len(P)))

    def gain_wait(self):
        """(info, gains): numpy copies of the context's pinned results, a GAIN_INFO_DTYPE record and VIEW_GAIN_DTYPE
        (n_views,).  A job on a field taken after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple
        as `.gain`."""
        pg = ctypes.c_void_p()
        info = np.zeros(1, GAIN_INFO_DTYPE)
        rc = self.lib.dsm_gain_wait(self.h, info.ctypes.data, ctypes.byref(pg))
        i = info[0]
        return self._waited(rc, "gain", lambda: (i, _take(pg, int(i["n_views"]), VIEW_GAIN_DTYPE)))

    # ---- viewpoints of frontier clusters against the latest known field ----
    def viewpoint_enable(self, max_clusters, max_candidates):
        self._ck(self.lib.dsm_viewpoint_enable(self.h, int(max_clusters), int(max_candidates)))

    def viewpoint_enqueue(self, camera, rotations, clusters, params):
        """camera: (fx, fy, cx, cy, width, height, max_range, unknown_blocks); rotations: (n, 9) row-major camera-to-world
        3x3 matrices; clusters: frontier-table indices; params: (r_min, r_max, dz_max, stride, max_samples, min_seen,
        top_k, with_reach, radius)."""
        self._viewpoint_enqueue(self.lib.dsm_viewpoint_enqueue, camera, rotations, clusters, params)

    def viewpoint_enqueue_terrain(self, camera, rotations, clusters, params, eye):
        """The viewpoint job on the plane of the latest terrain job (DESIGN.md §8.23), arguments as viewpoint_enqueue's
        with dz_max 0; the camera stands eye voxels above each candidate cell's support, and the slots' voxels that
        viewpoint_wait returns are cells q P + p of that plane."""
        self._viewpoint_enqueue(self.lib.dsm_viewpoint_enqueue_terrain, camera, rotations, clusters, params, int(eye))

    def _viewpoint_enqueue(self, call, camera, rotations, clusters, params, *eye):
        cam = _camera(camera)
        R = np.ascontiguousarray(rotations, np.float64).reshape(-1, 9)
        c = np.ascontiguousarray(clusters, np.int32).reshape(-1)
        p = DsmViewpointParams(*[int(x) for x in params[:8]], float(params[8]), 0)
        self._ck(call(self.h, ctypes.byref(cam), R.ctypes.data if len(R) else None, len(R), c.ctypes.data if len(c) else None, len(c),
                      ctypes.byref(p), *eye))

    def viewpoint_wait(self):
        """(info, clusters, viewpoints): numpy copies of the context's pinned results, a VIEWPOINT_INFO_DTYPE record,
        VIEWPOINT_CLUSTER_DTYPE (n_clusters,) and VIEWPOINT_DTYPE (n_clusters, top_k).  A job on a field taken after a
        rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.viewpoint`."""
        pc, pv = ctypes.c_void_p(), ctypes.c_void_p()
        info = np.zeros(1, VIEWPOINT_INFO_DTYPE)
        rc = self.lib.dsm_viewpoint_wait(self.h, info.ctypes.data, ctypes.byref(pc), ctypes.byref(pv))
        i = info[0]
        n, k = int(i["n_clusters"]), int(i["top_k"])
        return self._waited(rc, "viewpoint",
                            lambda: (i, _take(pc, n, VIEWPOINT_CLUSTER_DTYPE), _take(pv, n * k, VIEWPOINT_DTYPE).reshape(n, k)))

    # ---- the order of an exploration tour over a travel-cost matrix ----
    def tour_enable(self, max_sites, max_starts):
        self._ck(self.lib.dsm_tour_enable(self.h, int(max_sites), int(max_starts)))

    def tour_enqueue(self, matrix, open_, n_starts, max_passes, seed):
        """matrix: (n, n) uint32 costs, row i from site i (UINT32_MAX: no path), such as reach_matrix_wait's."""
        m = np.ascontiguousarray(matrix, np.uint32)
        if m.ndim != 2 or m.shape[0] != m.shape[1]:
            raise ValueError(f"a square matrix, not {m.shape}")
        self._ck(self.lib.dsm_tour_enqueue(self.h, m.ctypes.data if m.size else None, m.shape[0], int(open_), int(n_starts),
                                           int(max_passes), int(seed)))

    def tour_wait(self):
        """(info, starts, order): numpy copies of the context's pinned results, a TOUR_INFO_DTYPE record,
        TOUR_START_DTYPE (n_starts,) and the int32 order (n_sites,), -1 past n_included."""
        ps, po = ctypes.c_void_p(), ctypes.c_void_p()
        info = np.zeros(1, TOUR_INFO_DTYPE)
        self._ck(self.lib.dsm_tour_wait(self.h, info.ctypes.data, ctypes.byref(ps), ctypes.byref(po)))
        i = info[0]
        return i, _take(ps, int(i["n_starts"]), TOUR_START_DTYPE), _take(po, int(i["n_sites"]), np.int32)

    # ---- trajectory optimisation on the signed grid of the latest field ----
    def trajectory_enable(self, max_trajectories, max_points, max_memory):
        self._ck(self.lib.dsm_trajectory_enable(self.h, int(max_trajectories), int(max_points), int(max_memory)))

    def trajectory_enqueue(self, points, offsets, dt, params):
        """points (P, 3) float64 control points, offsets (n + 1,) int32, dt (n,) knot intervals; params a dict with the
        fields of DsmTrajectoryParams (reserved aside), such as oracle/pyoracle_trajectory.params() returns."""
        pts = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
        ofs = np.ascontiguousarray(offsets, np.int32).reshape(-1)
        dts = np.ascontiguousarray(dt, np.float64).reshape(-1)
        if len(ofs) < 2 or len(dts) != len(ofs) - 1:
            raise ValueError(f"{len(dts)} knot intervals for {max(len(ofs) - 1, 0)} trajectories")
        if not 0 <= ofs[-1] <= len(pts):
            raise ValueError(f"offsets end at {ofs[-1]}, beyond the {len(pts)} points")
        p = DsmTrajectoryParams(**{k: params[k] for k, _ in DsmTrajectoryParams._fields_ if k != "reserved"})
        self._ck(self.lib.dsm_trajectory_enqueue(self.h, pts.ctypes.data if len(pts) else None, ofs.ctypes.data if len(ofs) else None,
                                                 dts.ctypes.data if len(dts) else None, max(len(ofs) - 1, 0), ctypes.byref(p)))

    def trajectory_wait(self):
        """(info, records, points): numpy copies of the context's pinned results, a TRAJECTORY_INFO_DTYPE record,
        TRAJECTORY_DTYPE (n_trajectories,) and the optimised control points (n_points, 3).  A job on a field taken after a
        rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.trajectory`."""
        pr, pp = ctypes.c_void_p(), ctypes.c_void_p()
        info = np.zeros(1, TRAJECTORY_INFO_DTYPE)
        rc = self.lib.dsm_trajectory_wait(self.h, info.ctypes.data, ctypes.byref(pr), ctypes.byref(pp))
        i = info[0]
        n, n_pts = int(i["n_trajectories"]), int(i["n_points"])
        return self._waited(rc, "trajectory",
                            lambda: (i, _take(pr, n, TRAJECTORY_DTYPE), _take(pp, 3 * n_pts, np.float64).reshape(n_pts, 3)))

    # ---- headings along trajectories against the latest known field ----
    def heading_enable(self, max_trajectories, max_samples):
        self._ck(self.lib.dsm_heading_enable(self.h, int(max_trajectories), int(max_samples)))

    def heading_enqueue(self, points, offsets, camera, rotations, samples, requests, w_unknown, w_frontier):
        """points (P, 3) float64 control points and offsets (n + 1,) int32 as trajectory_enqueue takes them; camera:
        (fx, fy, cx, cy, width, height, max_range, unknown_blocks); rotations: (n_rot, 9) row-major camera-to-world 3x3
        matrices, neighbouring headings next to each other, cyclically; samples: K per segment; requests: n
        HEADING_REQUEST_DTYPE records or (start, end, max_step) rows; integer weights of the unknown and frontier counts."""
        pts = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
        ofs = np.ascontiguousarray(offsets, np.int32).reshape(-1)
        R = np.ascontiguousarray(rotations, np.float64).reshape(-1, 9)
        req = np.asarray(requests)
        if req.dtype != HEADING_REQUEST_DTYPE:
            rows = np.asarray(requests, np.int32).reshape(-1, 3)
            req = np.zeros(len(rows), HEADING_REQUEST_DTYPE)
            req["start"], req["end"], req["max_step"] = rows[:, 0], rows[:, 1], rows[:, 2]
        req = np.ascontiguousarray(req.reshape(-1))
        if len(ofs) < 2 or len(req) != len(ofs) - 1:
            raise ValueError(f"{len(req)} requests for {max(len(ofs) - 1, 0)} trajectories")
        if not 0 <= ofs[-1] <= len(pts):
            raise ValueError(f"offsets end at {ofs[-1]}, beyond the {len(pts)} points")
        cam = _camera(camera)
        self._ck(self.lib.dsm_heading_enqueue(self.h, pts.ctypes.data if len(pts) else None, ofs.ctypes.data, len(ofs) - 1,
                                              ctypes.byref(cam), R.ctypes.data if len(R) else None, len(R), int(samples),
                                              req.ctypes.data, int(w_unknown), int(w_frontier)))

    def heading_wait(self):
        """(info, records, samples, counts): numpy copies of the context's pinned results, a HEADING_INFO_DTYPE record,
        HEADING_DTYPE (n_trajectories,), HEADING_SAMPLE_DTYPE (n_samples,) and HEADING_COUNT_DTYPE (n_samples, n_rot).  A
        job on a field taken after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.heading`."""
        pr, ps, pc = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        info = np.zeros(1, HEADING_INFO_DTYPE)
        rc = self.lib.dsm_heading_wait(self.h, info.ctypes.data, ctypes.byref(pr), ctypes.byref(ps), ctypes.byref(pc))
        i = info[0]
        n, S, R = int(i["n_trajectories"]), int(i["n_samples"]), int(i["n_rot"])
        return self._waited(rc, "heading", lambda: (i, _take(pr, n, HEADING_DTYPE), _take(ps, S, HEADING_SAMPLE_DTYPE),
                                                    _take(pc, S * R, HEADING_COUNT_DTYPE).reshape(S, R)))

    # ---- the terrain of the latest known field ----
    def terrain_enable(self, up):
        """up in {+-1, +-2, +-3}: the field grid's axis |up| - 1, toward + or - (-2 for y-down camera frames)."""
        self._ck(self.lib.dsm_terrain_enable(self.h, int(up)))
        self._terrain_up = int(up)

    def terrain_enqueue(self, headroom, max_step):
        self._ck(self.lib.dsm_terrain_enqueue(self.h, int(headroom), int(max_step)))

    def terrain_wait(self):
        """(info, level, status, step, clearance): numpy copies of the context's pinned results, a TERRAIN_INFO_DTYPE
        record and the int16, uint8, uint8 and float32 planes [m2][m1][m0] of the terrain grid.  A job on a field taken
        after a rejected frame raises DsmError(DSM_E_CAPACITY) carrying the same tuple as `.terrain`."""
        pl, ps, pt, pc = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        info = np.zeros(1, TERRAIN_INFO_DTYPE)
        rc = self.lib.dsm_terrain_wait(self.h, info.ctypes.data, ctypes.byref(pl), ctypes.byref(ps), ctypes.byref(pt), ctypes.byref(pc))
        i = info[0]
        m0, m1, m2 = (int(x) for x in i["m"])
        cells = m0 * m1 * m2

        def planes():
            return (i,) + tuple(_take(p, cells, dt).reshape(m2, m1, m0) for p, dt in ((pl, np.int16), (ps, np.uint8), (pt, np.uint8),
                                                                                      (pc, np.float32)))
        return self._waited(rc, "terrain", planes)

    # ---- planner queries against the latest field ----
    def field_query_enable(self, max_points, max_trajectories, max_waypoints):
        self._ck(self.lib.dsm_field_query_enable(self.h, int(max_points), int(max_trajectories), int(max_waypoints)))

    def field_query_enqueue(self, points=None, waypoints=None, offsets=None, step=1.0, radius=0.0, signed=False):
        """points (n, 3) and trajectories (waypoints (w, 3), offsets (t + 1,), int32) as float64 / int32 arrays, either
        part may be None; step and radius in metres.  signed=True: dsm_field_query_enqueue_signed, on the signed grid."""
        pts = np.ascontiguousarray(np.zeros((0, 3)) if points is None else points, np.float64).reshape(-1, 3)
        wp = np.ascontiguousarray(np.zeros((0, 3)) if waypoints is None else waypoints, np.float64).reshape(-1, 3)
        ofs = np.ascontiguousarray(np.zeros(1) if offsets is None else offsets, np.int32).reshape(-1)
        n_traj = max(len(ofs) - 1, 0)
        fn = self.lib.dsm_field_query_enqueue_signed if signed else self.lib.dsm_field_query_enqueue
        self._ck(fn(self.h, pts.ctypes.data if len(pts) else None, len(pts), wp.ctypes.data if len(wp) else None,
                    ofs.ctypes.data if n_traj else None, n_traj, float(step), float(radius)))
        self._query_counts = (len(pts), n_traj)

    def field_query_wait(self):
        """(samples, clearance): numpy copies of the context's pinned results, FIELD_SAMPLE_DTYPE (n_points,) and
        CLEARANCE_DTYPE (n_trajectories,).  A query on a field taken after a rejected frame raises
        DsmError(DSM_E_CAPACITY) carrying the same tuple as `.query`."""
        ps, pc = ctypes.c_void_p(), ctypes.c_void_p()
        rc = self.lib.dsm_field_query_wait(self.h, ctypes.byref(ps), ctypes.byref(pc))

        def query():
            n_pts, n_traj = self._query_counts
            return _take(ps, n_pts, FIELD_SAMPLE_DTYPE), _take(pc, n_traj, CLEARANCE_DTYPE)
        return self._waited(rc, "query", query)

    # ---- raw cloud of a frame ----
    def frame_raw_cloud(self, frame, pose7, cap=None):
        """publish_raw_pointcloud (surfel_map.cpp:1115-1151) on frame `frame` of the most recent call that took images:
        W*H POINT_DTYPE points, column-major (point i*H + j = column i, row j).  pose7 = (px, py, pz, qx, qy, qz, qw)."""
        p = np.ascontiguousarray(pose7, dtype=np.float64).reshape(7)
        npx = self.cam.width * self.cam.height
        cap = npx if cap is None else cap
        return self._read(self.lib.dsm_frame_raw_cloud, POINT_DTYPE, cap, int(frame), _ptr(p))

    # ---- superpixel normal image of a frame ----
    def superpixel_image(self, frame=0, pitch=None):
        """FusionFunctions::debug_show (fusion_functions.cpp:977-1006) on frame `frame` of the most recent call that took
        images: [H][W][3] uint8, {|nx|, |ny|, |nz|} * 255 of each pixel's superpixel, black on label boundaries.
        `pitch` (bytes per row, >= 3*W) only sets the row pitch of the buffer the library writes into."""
        W, H = self.cam.width, self.cam.height
        pitch = 3 * W if pitch is None else int(pitch)
        buf = np.zeros((H, max(pitch, 1)), dtype=np.uint8)
        self._ck(self.lib.dsm_frame_superpixel_image(self.h, int(frame), _ptr(buf), pitch))
        return buf[:, :3 * W].reshape(H, W, 3).copy()

    # ---- parity readback ----
    def labels(self, frame=0):
        out = np.empty((self.cam.height, self.cam.width), dtype=np.int32)
        self._ck(self.lib.dsm_get_labels(self.h, frame, _ptr(out)))
        return out

    def seeds(self, frame=0):
        out = np.zeros(self.S, dtype=SEED_DTYPE)
        self._ck(self.lib.dsm_get_seeds(self.h, frame, _ptr(out)))
        return out

    def debug_stop_after(self, n):
        self._ck(self.lib.dsm_debug_stop_after(self.h, int(n)))

    def invariant_violations(self):
        c = ctypes.c_int(0)
        self._ck(self.lib.dsm_debug_invariant_violations(self.h, ctypes.byref(c)))
        return c.value

    # ---- measurement ----
    def profile_enable(self, mask):
        self._ck(self.lib.dsm_profile_enable(self.h, mask))

    def profile_reset(self):
        self._ck(self.lib.dsm_profile_reset(self.h))

    def profile_read(self):
        ms = np.zeros(NUM_KERNELS, dtype=np.float32)
        n = np.zeros(NUM_KERNELS, dtype=np.int32)
        self._ck(self.lib.dsm_profile_read(self.h, _ptr(ms), _ptr(n)))
        return ms, n

    def device_buffer(self, which):
        p = ctypes.c_void_p()
        sz = ctypes.c_size_t()
        self._ck(self.lib.dsm_device_buffer(self.h, which, ctypes.byref(p), ctypes.byref(sz)))
        return p.value, sz.value


class FusionFunctions:
    """Python mirror of the reference's `class FusionFunctions` public surface
    (fusion_functions.h:84-94): initialize(...) then fuse_initialize_map(...)."""

    def __init__(self, device=0, max_local_surfels=1 << 20):
        self._device = device
        self._cap = max_local_surfels
        self._ctx = None

    def initialize(self, width, height, fx, fy, cx, cy, fuse_far, fuse_near):
        from .synth import Camera
        self._ctx = Context(Camera(width, height, fx, fy, cx, cy, fuse_near, fuse_far),
                            max_batch=1, max_local_surfels=self._cap, device=self._device)

    def fuse_initialize_map(self, reference_frame_index, image, depth, pose, local_surfels):
        """Returns (local_surfels_updated, new_surfels) — the reference mutates the first in place
        and clears+fills the second (fusion_functions.cpp:30-83)."""
        if self._ctx is None:
            raise RuntimeError("initialize() has not been called")
        return self._ctx.fuse_frame(reference_frame_index, image, depth, pose, local_surfels)


# ---- output files (host only; no context, no GPU) ----
def _ck_io(rc, path):
    if rc != DSM_OK:
        raise DsmError(rc, f"{load_library().dsm_strerror(rc).decode()}: {path}")


def write_pcd(path, points, binary=False):
    """SurfelMap::save_cloud's file (surfel_map.cpp:1171): PCD v0.7 with fields x y z intensity."""
    points = np.ascontiguousarray(points, dtype=POINT_DTYPE)
    _ck_io(load_library().dsm_write_pcd(os.fsencode(path), _ptr(points) if len(points) else None, len(points), int(binary)), path)


def write_ply_mesh(path, surfels):
    """SurfelMap::save_mesh (surfel_map.cpp:1229-1280): one hexagon per surfel, ASCII PLY."""
    surfels = np.ascontiguousarray(surfels, dtype=SURFEL_DTYPE)
    _ck_io(load_library().dsm_write_ply_mesh(os.fsencode(path), _ptr(surfels) if len(surfels) else None, len(surfels)), path)


def map_peek(path):
    """(extra bytes, segment table [n, 3]) of a checkpoint file, checked without a context."""
    L = load_library()
    ne, ns = ctypes.c_size_t(0), ctypes.c_int(0)
    _ck_io(L.dsm_map_peek(os.fsencode(path), None, 0, ctypes.byref(ne), None, 0, ctypes.byref(ns)), path)
    extra = ctypes.create_string_buffer(max(ne.value, 1))
    seg = np.zeros((max(ns.value, 1), 3), np.int32)
    _ck_io(L.dsm_map_peek(os.fsencode(path), extra, ne.value, None, _ptr(seg), ns.value, None), path)
    return extra.raw[:ne.value], seg[:ns.value].copy()


def map_peek_journal(path):
    """(extra bytes, segment table [n, 3], records applied) of the state base + journal resolve to, without a context."""
    L = load_library()
    ne, ns, rec = ctypes.c_size_t(0), ctypes.c_int(0), ctypes.c_int(0)
    _ck_io(L.dsm_map_peek_journal(os.fsencode(path), None, 0, ctypes.byref(ne), None, 0, ctypes.byref(ns), None), path)
    extra = ctypes.create_string_buffer(max(ne.value, 1))
    seg = np.zeros((max(ns.value, 1), 3), np.int32)
    _ck_io(L.dsm_map_peek_journal(os.fsencode(path), extra, ne.value, None, _ptr(seg), ns.value, None, ctypes.byref(rec)), path)
    return extra.raw[:ne.value], seg[:ns.value].copy(), rec.value


def journal_materialize(path, out_path):
    """The version-1 checkpoint file of the state base + journal resolve to, written to out_path."""
    _ck_io(load_library().dsm_journal_materialize(os.fsencode(path), os.fsencode(out_path)), path)


def mesh_vertices(surfels):
    """push_a_surfel (surfel_map.cpp:1175-1226): float32 [n, 6, 6] = 6 vertices x (x, y, z, c, c, c)."""
    surfels = np.ascontiguousarray(surfels, dtype=SURFEL_DTYPE)
    out = np.zeros((len(surfels), 6, 6), dtype=np.float32)
    _ck_io(load_library().dsm_mesh_vertices(_ptr(surfels) if len(surfels) else None, len(surfels), _ptr(out) if len(surfels) else None), "")
    return out
