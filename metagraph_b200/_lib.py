"""ctypes binding of the C-ABI in include/mgb.h.

The product library is metagraph_b200/_lib/libmgb.so (built by __graft_entry__.build() with nvcc
for sm_90a, H100). There is no CPU implementation: if the library is missing, loading fails.
"""
import ctypes
import os

from .config import mgb_config_t

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "_lib", "libmgb.so")

MGB_OK = 0
ERRORS = {-1: "INVALID_ARGUMENT", -2: "CUDA", -3: "BAD_CONFIG", -4: "UNSUPPORTED", -5: "OVERFLOW",
          -6: "NO_DEVICE", -7: "NO_MEMORY"}


class MgbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("mgb error %d (%s): %s" % (code, ERRORS.get(code, "?"), msg))
        self.code = code


class mgb_alignment_t(ctypes.Structure):
    _fields_ = [
        ("read_index", ctypes.c_uint32), ("orientation", ctypes.c_uint8), ("pad", ctypes.c_uint8 * 3),
        ("score", ctypes.c_int32), ("offset", ctypes.c_uint32), ("query_begin", ctypes.c_uint32),
        ("query_len", ctypes.c_uint32), ("num_nodes", ctypes.c_uint32), ("sequence_len", ctypes.c_uint32),
        ("num_cigar_ops", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
        ("nodes", ctypes.POINTER(ctypes.c_uint64)), ("sequence", ctypes.POINTER(ctypes.c_char)),
        ("cigar", ctypes.POINTER(ctypes.c_uint32)),
    ]


class mgb_stats_t(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in
                ("num_seeds", "num_extensions", "num_explored_nodes", "dp_cells", "dp_columns",
                 "num_reads_retried")] + \
               [(n, ctypes.c_double) for n in ("seed_kernel_ms", "align_kernel_ms", "h2d_ms", "d2h_ms")] + \
               [(n, ctypes.c_uint64) for n in ("h2d_bytes", "d2h_bytes", "kernel_launches")]


class mgb_device_sizes_t(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in ("n_reads", "n_alignments", "sequence_bytes", "cigar_ops", "nodes")]


# mgb_device_columns_t: device pointers, in the order of include/mgb.h
DEVICE_COLUMNS = ("read_first", "read_index", "orientation", "score", "offset", "query_begin", "query_len", "num_nodes",
                  "sequence_len", "num_cigar_ops", "sequence", "sequence_offsets", "cigar", "cigar_offsets", "nodes",
                  "node_offsets")


class mgb_device_columns_t(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in DEVICE_COLUMNS]


class mgb_boss_t(ctypes.Structure):
    _fields_ = [("n_plus_1", ctypes.c_uint64), ("W", ctypes.POINTER(ctypes.c_uint8)),
                ("last", ctypes.POINTER(ctypes.c_uint8)), ("F", ctypes.c_uint64 * 32),
                ("k", ctypes.c_uint32), ("alphabet", ctypes.c_int32)]


_libs = {}


def load_library(path=None):
    # MGB_LIB: another build of the same library (e.g. one with phase timers), for probes
    path = os.path.abspath(path or os.environ.get("MGB_LIB") or DEFAULT_LIB)
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise ImportError(
            "%s not found: build the sm_90a extension first (python -c 'import __graft_entry__ as g; "
            "g.build()'). metagraph_b200 has no CPU fallback." % path)
    L = ctypes.CDLL(path)
    u64, u32, vp, cp, i = ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int
    L.mgb_last_error.restype = cp
    L.mgb_device_count.restype = i
    L.mgb_index_create.restype = i
    L.mgb_index_create.argtypes = [vp, vp, u64, vp, vp, u32, i, u32, i, ctypes.POINTER(vp)]
    L.mgb_index_destroy.argtypes = [vp]
    L.mgb_index_num_edges.restype = u64
    L.mgb_index_num_edges.argtypes = [vp]
    L.mgb_index_device_bytes.restype = u64
    L.mgb_index_device_bytes.argtypes = [vp]
    L.mgb_index_k.restype = u32
    L.mgb_index_k.argtypes = [vp]
    L.mgb_config_init.argtypes = [ctypes.POINTER(mgb_config_t)]
    L.mgb_config_init_cli.argtypes = [ctypes.POINTER(mgb_config_t), u32, i]
    L.mgb_config_check.restype = i
    L.mgb_config_check.argtypes = [vp, ctypes.POINTER(mgb_config_t)]
    L.mgb_map_to_nodes.restype = i
    L.mgb_map_to_nodes.argtypes = [vp, vp, vp, u32, vp]
    L.mgb_map_to_nodes_strands.restype = i
    L.mgb_map_to_nodes_strands.argtypes = [vp, vp, vp, u32, vp, vp]
    L.mgb_align_batch.restype = i
    L.mgb_align_batch.argtypes = [vp, ctypes.POINTER(mgb_config_t), vp, vp, u32, ctypes.POINTER(vp)]
    L.mgb_align_batch_text.restype = i
    L.mgb_align_batch_text.argtypes = [vp, ctypes.POINTER(mgb_config_t), vp, vp, vp, vp, u32, i, ctypes.POINTER(vp)]
    L.mgb_align_fastx_text.restype = i
    L.mgb_align_fastx_text.argtypes = [vp, ctypes.POINTER(mgb_config_t), vp, u64, i, cp, i, i, ctypes.POINTER(u64),
                                       ctypes.POINTER(i), ctypes.POINTER(vp)]
    L.mgb_index_replicate.restype = i
    L.mgb_index_replicate.argtypes = [vp, i, ctypes.POINTER(vp)]
    L.mgb_fastx_stage.restype = i
    L.mgb_fastx_stage.argtypes = [vp, vp, u64, i, cp, i, ctypes.POINTER(u64), ctypes.POINTER(i), ctypes.POINTER(vp)]
    L.mgb_align_fastx_batch_text.restype = i
    L.mgb_align_fastx_batch_text.argtypes = [vp, ctypes.POINTER(mgb_config_t), vp, i, ctypes.POINTER(vp)]
    L.mgb_fastx_batch_free.restype = None
    L.mgb_fastx_batch_free.argtypes = [vp]
    L.mgb_fastx_stage_bgzf.restype = i
    L.mgb_fastx_stage_bgzf.argtypes = [vp, vp, u64, vp, u64, i, u64, cp, i, ctypes.POINTER(u64), ctypes.POINTER(i),
                                       ctypes.POINTER(u64), ctypes.POINTER(i), ctypes.POINTER(vp)]
    L.mgb_fastx_batch_tail.restype = i
    L.mgb_fastx_batch_tail.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(u64)]
    L.mgb_bgzf_inflate.restype = i
    L.mgb_bgzf_inflate.argtypes = [vp, vp, u64, i, vp, u64, ctypes.POINTER(u64), ctypes.POINTER(u64),
                                   ctypes.POINTER(u64), ctypes.POINTER(i)]
    L.mgb_gzip_stream_create.restype = i
    L.mgb_gzip_stream_create.argtypes = [ctypes.POINTER(vp)]
    L.mgb_gzip_stream_free.restype = None
    L.mgb_gzip_stream_free.argtypes = [vp]
    L.mgb_gzip_stream_state.restype = i
    L.mgb_gzip_stream_state.argtypes = [vp, ctypes.POINTER(i), ctypes.POINTER(u64)]
    L.mgb_gzip_stream_export_bytes.restype = u64
    L.mgb_gzip_stream_export_bytes.argtypes = [vp]
    L.mgb_gzip_stream_export.restype = i
    L.mgb_gzip_stream_export.argtypes = [vp, vp, u64]
    L.mgb_gzip_stream_import.restype = i
    L.mgb_gzip_stream_import.argtypes = [vp, u64, ctypes.POINTER(vp)]
    L.mgb_fastx_stage_gzip.restype = i
    L.mgb_fastx_stage_gzip.argtypes = [vp, vp, vp, u64, vp, u64, i, u64, cp, i, ctypes.POINTER(u64), ctypes.POINTER(i),
                                       ctypes.POINTER(u64), ctypes.POINTER(i), ctypes.POINTER(vp)]
    L.mgb_gzip_inflate.restype = i
    L.mgb_gzip_inflate.argtypes = [vp, vp, u64, i, u64, vp, u64, vp, u64, ctypes.POINTER(u64), ctypes.POINTER(u64),
                                   ctypes.POINTER(i), vp]
    L.mgb_fastx_parse.restype = i
    L.mgb_fastx_parse.argtypes = [vp, vp, u64, i, cp, i, i, vp, u64, vp, vp, u64, vp, u64, ctypes.POINTER(u64),
                                  ctypes.POINTER(u64), ctypes.POINTER(i), ctypes.POINTER(i)]
    L.mgb_results_text.restype = i
    L.mgb_results_text.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(u64)]
    L.mgb_results_num_reads.restype = u32
    L.mgb_results_num_reads.argtypes = [vp]
    L.mgb_results_read_range.argtypes = [vp, u32, ctypes.POINTER(u64), ctypes.POINTER(u32)]
    L.mgb_results_num_alignments.restype = u64
    L.mgb_results_num_alignments.argtypes = [vp]
    L.mgb_results_alignments.restype = ctypes.POINTER(mgb_alignment_t)
    L.mgb_results_alignments.argtypes = [vp]
    L.mgb_results_stats.restype = ctypes.POINTER(mgb_stats_t)
    L.mgb_results_stats.argtypes = [vp]
    L.mgb_results_free.argtypes = [vp]
    L.mgb_results_export_bytes.restype = u64
    L.mgb_results_export_bytes.argtypes = [vp]
    L.mgb_results_export.restype = i
    L.mgb_results_export.argtypes = [vp, vp, u64]
    L.mgb_results_import.restype = i
    L.mgb_results_import.argtypes = [vp, u64, u32, ctypes.POINTER(vp)]
    L.mgb_boss_build.restype = i
    L.mgb_boss_build.argtypes = [vp, vp, u32, u32, i, i, i, ctypes.POINTER(mgb_boss_t)]
    L.mgb_boss_free.argtypes = [ctypes.POINTER(mgb_boss_t)]
    L.mgb_boss_mask_dummy.restype = i
    L.mgb_boss_mask_dummy.argtypes = [ctypes.POINTER(mgb_boss_t), vp]
    L.mgb_index_set_mode.restype = i
    L.mgb_index_set_mode.argtypes = [vp, i]
    L.mgb_dbg_load.restype = i
    L.mgb_dbg_load.argtypes = [ctypes.c_char_p, ctypes.POINTER(mgb_boss_t), ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    L.mgb_dbg_last_error.restype = ctypes.c_char_p
    L.mgb_boss_last_error.restype = ctypes.c_char_p
    L.mgb_set_pipeline_pieces.restype = None
    L.mgb_set_pipeline_pieces.argtypes = [u32]
    L.mgb_set_host_threads.restype = None
    L.mgb_align_batch_device.restype = i
    L.mgb_align_batch_device.argtypes = [vp, ctypes.POINTER(mgb_config_t), vp, vp, i, u32, vp, ctypes.POINTER(vp)]
    L.mgb_device_results_sizes.restype = i
    L.mgb_device_results_sizes.argtypes = [vp, ctypes.POINTER(mgb_device_sizes_t)]
    L.mgb_device_results_stats.restype = ctypes.POINTER(mgb_stats_t)
    L.mgb_device_results_stats.argtypes = [vp]
    L.mgb_device_results_write.restype = i
    L.mgb_device_results_write.argtypes = [vp, ctypes.POINTER(mgb_device_columns_t), vp]
    L.mgb_device_results_free.restype = None
    L.mgb_device_results_free.argtypes = [vp]
    L.mgb_set_host_threads.argtypes = [i]
    _libs[path] = L
    return L


def check(L, rc):
    if rc != MGB_OK:
        raise MgbError(rc, L.mgb_last_error().decode())


REQUIRED_SYMBOLS = [
    "mgb_last_error", "mgb_device_count", "mgb_index_create", "mgb_index_destroy", "mgb_index_num_edges",
    "mgb_index_device_bytes", "mgb_index_k", "mgb_config_init", "mgb_config_init_cli", "mgb_map_to_nodes",
    "mgb_map_to_nodes_strands",    "mgb_align_batch", "mgb_results_num_reads", "mgb_results_read_range", "mgb_results_num_alignments",
    "mgb_results_alignments", "mgb_results_stats", "mgb_results_free", "mgb_results_export_bytes",
    "mgb_results_export", "mgb_results_import", "mgb_boss_build", "mgb_boss_free",
    "mgb_boss_mask_dummy", "mgb_set_pipeline_pieces", "mgb_set_host_threads", "mgb_dbg_load", "mgb_dbg_last_error", "mgb_boss_last_error", "mgb_config_check", "mgb_dbg_load_suffix_ranges", "mgb_dbg_free_suffix_ranges", "mgb_index_set_mode",
    "mgb_align_batch_text", "mgb_results_text", "mgb_align_fastx_text", "mgb_fastx_parse", "mgb_index_replicate",
    "mgb_fastx_stage", "mgb_align_fastx_batch_text", "mgb_fastx_batch_free", "mgb_fastx_stage_bgzf",
    "mgb_fastx_batch_tail", "mgb_bgzf_inflate", "mgb_gzip_stream_create", "mgb_gzip_stream_free",
    "mgb_gzip_stream_state", "mgb_fastx_stage_gzip", "mgb_gzip_inflate", "mgb_gzip_stream_export_bytes",
    "mgb_gzip_stream_export", "mgb_gzip_stream_import", "mgb_align_batch_device", "mgb_device_results_sizes",
    "mgb_device_results_stats", "mgb_device_results_write", "mgb_device_results_free",
]
MGB_TEXT_TSV, MGB_TEXT_JSON = 1, 2
MGB_FASTX_FWD_AND_REVERSE = 1
