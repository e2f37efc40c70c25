"""ctypes binding of the C ABI declared in include/simdjson_b200.h.

The shared library is built in-tree by __graft_entry__.build() (nvcc, sm_90a) as
simdjson-go_b200/libsimdjson_b200.so.  There is no CPU fallback: loading fails loudly if
the library is missing, and every call fails with SJ_ERR_NO_DEVICE without an H100.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SJ_B200_LIB") or os.path.join(os.path.dirname(_HERE), "libsimdjson_b200.so")  # override: another build, e.g. to compare two

ERR_EXCHANGE, ERR_PEER, ERR_UNSUPPORTED, EXCHANGE_HANDLE_BYTES = 10, 11, 12, 64
FLAG_NDJSON = 1
FLAG_COPY_STRINGS = 2
OK, ERR_STAGE1, ERR_STAGE2, ERR_NO_DEVICE, ERR_CAPACITY, ERR_TOO_LARGE, ERR_ARGUMENT = range(7)

# every symbol include/simdjson_b200.h declares
EXPORTS = [
    "sj_supported", "sj_device_count", "sj_error_string", "sj_ctx_create", "sj_ctx_destroy", "sj_ctx_set_stage2_impl", "sj_ctx_set_stream", "sj_bind_to_device_numa", "sj_host_alloc",
    "sj_host_free", "sj_trim_space", "sj_bounds", "sj_parse", "sj_parse_device", "sj_gen_ndjson_device", "sj_parse_nd_sharded_count", "sj_parse_nd_sharded_emit", "sj_exchange_create", "sj_exchange_set_gap", "sj_exchange_set_timeout_ms", "sj_exchange_connect", "sj_exchange_connect_ptrs", "sj_exchange_local", "sj_exchange_bases", "sj_exchange_result", "sj_find_structural_indices", "sj_stage1_device",
    "sj_stage1_launch", "sj_ctx_sync", "sj_event_record", "sj_event_elapsed_ms", "sj_kernel_launches",
    "sj_test_block_masks", "sj_test_geometry", "sj_test_finalize", "sj_test_flatten_bits", "sj_test_parse_strings",
    "sj_test_parse_numbers", "sj_count_where_device", "sj_parse_count_where", "sj_marshal_device", "sj_parse_marshal", "sj_serialize_device", "sj_parse_serialize",
    "sj_deserialize_device", "sj_test_set_string_hash_bits", "sj_test_stage2_internal", "sj_stream_create", "sj_stream_destroy",
    "sj_stream_write", "sj_stream_close_input", "sj_stream_next", "sj_stream_release",
]
STREAM_END, STREAM_EMPTY, STREAM_BUSY = 7, 8, 9


class StreamResult(C.Structure):
    _fields_ = [("message", C.c_void_p), ("message_len", C.c_size_t), ("tape", C.c_void_p), ("tape_len", C.c_size_t),
                ("strings", C.c_void_p), ("strings_len", C.c_size_t), ("seq", C.c_uint64), ("slot", C.c_void_p)]


class ShardTotals(C.Structure):
    _fields_ = [("msg_bytes", C.c_uint64), ("tape_words", C.c_uint64), ("string_bytes", C.c_uint64), ("records", C.c_uint64)]


class Stage1Info(C.Structure):
    _fields_ = [("n_idx", C.c_uint64), ("error", C.c_uint32), ("ends_in_string", C.c_uint32),
                ("last_pos", C.c_uint32), ("overflow", C.c_uint32)]


_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("simdjson_b200: %s is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a); there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, sz, u32, u64, i32 = C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64, C.c_int
    szp = C.POINTER(C.c_size_t)
    L.sj_supported.restype = i32
    L.sj_device_count.restype = i32
    L.sj_error_string.restype = C.c_char_p
    L.sj_error_string.argtypes = [i32]
    L.sj_ctx_create.restype = i32
    L.sj_ctx_create.argtypes = [i32, C.POINTER(vp)]
    L.sj_ctx_destroy.restype = None
    L.sj_ctx_destroy.argtypes = [vp]
    L.sj_ctx_set_stage2_impl.restype = i32
    L.sj_ctx_set_stage2_impl.argtypes = [vp, i32]
    L.sj_test_geometry.restype = None
    L.sj_test_geometry.argtypes = [vp]
    L.sj_host_alloc.restype = vp
    L.sj_host_alloc.argtypes = [sz]
    L.sj_host_free.restype = None
    L.sj_host_free.argtypes = [vp]
    L.sj_trim_space.restype = None
    L.sj_trim_space.argtypes = [vp, sz, szp, szp]
    L.sj_bounds.restype = None
    L.sj_bounds.argtypes = [sz, szp, szp]
    L.sj_parse.restype = i32
    L.sj_parse.argtypes = [vp, vp, sz, u32, vp, sz, szp, vp, sz, szp, szp, szp]
    L.sj_parse_device.restype = i32
    L.sj_parse_device.argtypes = [vp, vp, sz, u32, vp, sz, szp, vp, sz, szp]
    L.sj_parse_nd_sharded_count.restype = i32
    L.sj_parse_nd_sharded_count.argtypes = [vp, vp, sz, u32, C.POINTER(ShardTotals), vp]
    L.sj_parse_nd_sharded_emit.restype = i32
    L.sj_parse_nd_sharded_emit.argtypes = [vp, C.c_uint64, C.c_uint64, C.c_uint64, vp, vp, sz, vp, sz]
    L.sj_exchange_create.restype = i32
    L.sj_exchange_create.argtypes = [vp, i32, i32, C.c_uint64, vp]
    L.sj_exchange_set_gap.restype = i32
    L.sj_exchange_set_gap.argtypes = [vp, C.c_uint64]
    L.sj_exchange_set_timeout_ms.restype = i32
    L.sj_exchange_set_timeout_ms.argtypes = [vp, u32]
    L.sj_exchange_connect.restype = i32
    L.sj_exchange_connect.argtypes = [vp, vp]
    L.sj_exchange_connect_ptrs.restype = i32
    L.sj_exchange_connect_ptrs.argtypes = [vp, C.POINTER(vp)]
    L.sj_exchange_local.restype = vp
    L.sj_exchange_local.argtypes = [vp]
    L.sj_exchange_bases.restype = vp
    L.sj_exchange_bases.argtypes = [vp]
    L.sj_exchange_result.restype = i32
    L.sj_exchange_result.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.sj_gen_ndjson_device.restype = i32
    L.sj_gen_ndjson_device.argtypes = [vp, vp, sz, C.c_uint64, C.c_uint64, vp, sz, szp]
    L.sj_bind_to_device_numa.restype = i32
    L.sj_bind_to_device_numa.argtypes = [i32]
    L.sj_ctx_set_stream.restype = i32
    L.sj_ctx_set_stream.argtypes = [vp, vp]
    L.sj_find_structural_indices.restype = i32
    L.sj_find_structural_indices.argtypes = [vp, vp, sz, i32, vp, sz, szp]
    L.sj_stage1_device.restype = i32
    L.sj_stage1_device.argtypes = [vp, vp, sz, i32, i32, vp, sz, C.POINTER(Stage1Info)]
    L.sj_stage1_launch.restype = i32
    L.sj_stage1_launch.argtypes = [vp, vp, sz, i32, i32, vp, sz]
    L.sj_ctx_sync.restype = i32
    L.sj_ctx_sync.argtypes = [vp]
    L.sj_event_record.restype = i32
    L.sj_event_record.argtypes = [vp, i32]
    L.sj_event_elapsed_ms.restype = i32
    L.sj_event_elapsed_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.sj_kernel_launches.restype = i32
    L.sj_kernel_launches.argtypes = [vp, C.POINTER(u64)]
    L.sj_test_block_masks.restype = i32
    L.sj_test_block_masks.argtypes = [vp, vp, sz, vp, vp]
    L.sj_test_finalize.restype = i32
    L.sj_test_finalize.argtypes = [vp, vp, sz, vp]
    L.sj_test_flatten_bits.restype = i32
    L.sj_test_flatten_bits.argtypes = [vp, vp, sz, vp, sz, szp]
    L.sj_test_parse_strings.restype = i32
    L.sj_test_parse_strings.argtypes = [vp, vp, vp, sz, vp, vp, vp, vp, vp]
    L.sj_test_parse_numbers.restype = i32
    L.sj_test_parse_numbers.argtypes = [vp, vp, vp, sz, vp, vp]
    L.sj_count_where_device.restype = i32
    L.sj_count_where_device.argtypes = [vp, vp, vp, sz, vp, C.c_char_p, sz, C.c_char_p, sz, C.POINTER(u64), C.POINTER(u64)]
    L.sj_parse_count_where.restype = i32
    L.sj_parse_count_where.argtypes = [vp, vp, sz, u32, C.c_char_p, sz, C.c_char_p, sz, C.POINTER(u64), C.POINTER(u64)]
    L.sj_marshal_device.restype = i32
    L.sj_marshal_device.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, szp]
    L.sj_parse_marshal.restype = i32
    L.sj_parse_marshal.argtypes = [vp, vp, sz, u32, vp, sz, szp]
    L.sj_serialize_device.restype = i32
    L.sj_serialize_device.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, szp]
    L.sj_parse_serialize.restype = i32
    L.sj_parse_serialize.argtypes = [vp, vp, sz, u32, vp, sz, szp]
    L.sj_deserialize_device.restype = i32
    L.sj_deserialize_device.argtypes = [vp, vp, sz, vp, sz, szp, vp, sz, szp, vp, sz, szp]
    L.sj_test_set_string_hash_bits.restype = i32
    L.sj_test_set_string_hash_bits.argtypes = [vp, i32]
    L.sj_test_stage2_internal.restype = i32
    L.sj_test_stage2_internal.argtypes = [vp, C.POINTER(u32)]
    L.sj_stream_create.restype = i32
    L.sj_stream_create.argtypes = [i32, i32, sz, u32, C.POINTER(vp)]
    L.sj_stream_destroy.restype = None
    L.sj_stream_destroy.argtypes = [vp]
    L.sj_stream_write.restype = i32
    L.sj_stream_write.argtypes = [vp, vp, sz, szp]
    L.sj_stream_close_input.restype = i32
    L.sj_stream_close_input.argtypes = [vp]
    L.sj_stream_next.restype = i32
    L.sj_stream_next.argtypes = [vp, C.POINTER(StreamResult)]
    L.sj_stream_release.restype = i32
    L.sj_stream_release.argtypes = [vp, C.POINTER(StreamResult)]
    _lib = L
    return L


class SjError(RuntimeError):
    def __init__(self, rc):
        self.rc = rc
        msg = load().sj_error_string(rc)
        super().__init__("simdjson_b200: rc=%d (%s)" % (rc, msg.decode() if msg else "?"))
