"""ctypes binding of include/b2rpc.h (brpc_b200/libb2rpc.so)."""
import atexit
import ctypes as C
import gc
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
lib_path = os.environ.get("B2RPC_LIB") or os.path.join(_HERE, "libb2rpc.so")      # (B2RPC_LIB: A/B builds of the same library for tuning runs)

B2_OK, B2_E_INVAL, B2_E_NO_DEVICE, B2_E_CUDA, B2_E_CAPACITY, B2_E_NOMEM = 0, -1, -2, -3, -4, -5

RUN_DT = np.dtype([("socket_id", "<u8"), ("offset", "<u4"), ("length", "<u4"),
                   ("preferred_proto", "<i4"), ("flags", "<u4")])
RUN_STATUS_DT = np.dtype([("consumed", "<u4"), ("parse_error", "<u4"), ("n_msgs", "<u4"), ("first_msg", "<u4"),
                          ("preferred_proto", "<i4"), ("n_unanswered", "<u4"), ("resp_off", "<u4"), ("resp_bytes", "<u4")])
H2_FRAME_DT = np.dtype([("type", "u1"), ("flags", "u1"), ("pad", "<u2"), ("stream_id", "<u4"), ("payload_off", "<u4"), ("payload_len", "<u4")])
HPACK_BLOCK_DT = np.dtype([("conn", "<u4"), ("offset", "<u4"), ("length", "<u4"), ("reserved", "<u4")])
H2_RUN_STATUS_DT = np.dtype([("consumed", "<u4"), ("parse_error", "<u4"), ("n_msgs", "<u4"), ("first_msg", "<u4"), ("ctrl_off", "<u4"), ("ctrl_len", "<u4"),
                             ("remote_max_frame_size", "<u4"), ("remote_stream_window_size", "<u4")])
REQUEST_DT = np.dtype([("kind", "<u4"), ("flags", "<u4"), ("method_idx", "<i4"), ("timeout_ms", "<i4"), ("correlation_id", "<i8"), ("log_id", "<i8"),
                       ("compress_type", "<i4"), ("checksum_type", "<i4"), ("frame_type", "<i4"), ("payload_off", "<u4"), ("payload_len", "<u4"),
                       ("attachment_off", "<u4"), ("attachment_len", "<u4"), ("reserved", "<u4")])
REPLY_DT = np.dtype([("flags", "<u4"), ("error_code", "<i4"), ("correlation_id", "<i8"), ("compress_type", "<i4"), ("checksum_type", "<i4"),
                     ("content_type", "<i4"), ("error_text_off", "<u4"), ("error_text_len", "<u4"), ("body_off", "<u4"), ("body_len", "<u4"),
                     ("attachment_off", "<u4"), ("attachment_len", "<u4"), ("checksum_value_off", "<u4"), ("checksum_value_len", "<u4"),
                     ("extra_streams_off", "<u4"), ("n_extra_streams", "<u4"), ("user_fields_off", "<u4"), ("n_user_fields", "<u4"),
                     ("reserved", "<u4"), ("stream_id", "<i8")])          # == b2_reply, 88 bytes
H2_RESPONSE_DT = np.dtype([("conn", "<u4"), ("stream_id", "<u4"), ("status_code", "<i4"), ("flags", "<u4"), ("content_type_off", "<u4"),
                           ("content_type_len", "<u4"), ("body_off", "<u4"), ("body_len", "<u4"), ("grpc_status", "<i4"),
                           ("grpc_message_off", "<u4"), ("grpc_message_len", "<u4"), ("reserved", "<u4")])
H2_REQUEST_DT = np.dtype([("conn", "<u4"), ("flags", "<u4"), ("path_off", "<u4"), ("path_len", "<u4"), ("authority_off", "<u4"),
                          ("authority_len", "<u4"), ("content_type_off", "<u4"), ("content_type_len", "<u4"), ("body_off", "<u4"),
                          ("body_len", "<u4"), ("extra_off", "<u4"), ("extra_len", "<u4")])          # == b2_h2_request, 48 bytes
H2_PEER_UPDATE_DT = np.dtype([("set", "<u4"), ("header_table_size", "<u4"), ("max_frame_size", "<u4"), ("stream_window_size", "<u4"), ("conn_window_add", "<i8")])
H2_REQUEST_RESULT_DT = np.dtype([("status", "<i4"), ("stream_id", "<u4"), ("out_off", "<u4"), ("out_len", "<u4")])
H2_MSG_DT = np.dtype([("run_idx", "<u4"), ("stream_id", "<u4"), ("headers_off", "<u4"), ("headers_len", "<u4"), ("n_headers", "<u4"),
                      ("body_off", "<u4"), ("body_len", "<u4"), ("http_method", "<u4"), ("content_type", "<u4"), ("flags", "<u4"),
                      ("method_idx", "<i4"), ("msg_off", "<u4"), ("msg_len", "<u4"), ("path_off", "<u4"), ("path_len", "<u4"), ("reserved", "<u4")])
H2_CALL_DT = np.dtype([("run_idx", "<u4"), ("stream_id", "<u4"), ("how", "<u4"), ("status_code", "<i4"), ("error_code", "<i4"), ("grpc_status", "<i4"),
                       ("headers_off", "<u4"), ("headers_len", "<u4"), ("n_headers", "<u4"), ("body_off", "<u4"), ("body_len", "<u4"),
                       ("msg_off", "<u4"), ("msg_len", "<u4"), ("error_off", "<u4"), ("error_len", "<u4"), ("flags", "<u4")])   # == b2_h2_call, 64 bytes
# b2_h2_msg / b2_h2_call flags of connections opted in with Context.h2_conn_set_gunzip (include/b2rpc.h)
H2_FLAG_GUNZIPPED, H2_FLAG_GUNZIP_HOST, H2_FLAG_NO_GRPC_ENCODING = 64, 128, 256
# b2_h2_msg flag of a call Context.h2_serve_batch answered on the device (msgs["reserved"] then holds the reply's grpc-status)
H2_FLAG_ANSWERED = 512
H2_REPLY_SPAN_DT = np.dtype([("off", "<u4"), ("len", "<u4"), ("n_answered", "<u4"), ("reserved", "<u4")])   # == b2_h2_reply_span, 16 bytes
MSG_DT = np.dtype([("run_idx", "<u4"), ("frame_off", "<u4"), ("body_size", "<u4"), ("meta_size", "<u4"),
                   ("correlation_id", "<i8"), ("log_id", "<i8"),
                   ("attachment_size", "<i4"), ("compress_type", "<i4"), ("checksum_type", "<i4"), ("error_code", "<i4"),
                   ("has_bits", "<u2"), ("protocol", "u1"), ("content_type", "u1"),
                   ("method_idx", "<i2"), ("status", "<u2"), ("resp_off", "<u4"), ("resp_len", "<u4")])
assert RUN_DT.itemsize == 24 and RUN_STATUS_DT.itemsize == 32 and MSG_DT.itemsize == 64
# the stream table (b2_stream_*)
STREAM_DESC_DT = np.dtype([("stream_id", "<i8"), ("remote_stream_id", "<i8"), ("host_socket_id", "<u8"), ("flags", "<u4"), ("max_buf_size", "<u4")])
STREAM_MSG_DT = np.dtype([("stream_id", "<i8"), ("first_frame", "<u4"), ("n_frames", "<u4"), ("off", "<u4"), ("len", "<u4"), ("flags", "<u4"), ("reserved", "<u4")])
STREAM_EVENT_DT = np.dtype([("stream_id", "<i8"), ("host_socket_id", "<u8"), ("local_consumed", "<u8"), ("remote_consumed", "<u8"), ("n_msgs", "<u4"),
                            ("first_msg", "<u4"), ("consumed_bytes", "<u4"), ("flags", "<u4"), ("fb_off", "<u4"), ("fb_len", "<u4"), ("close_off", "<u4"),
                            ("close_len", "<u4"), ("handover_msg", "<u4"), ("pending_bytes", "<u4"), ("reserved", "<u4", (2,))])
assert STREAM_DESC_DT.itemsize == 32 and STREAM_MSG_DT.itemsize == 32 and STREAM_EVENT_DT.itemsize == 80
STREAM_CONNECTED, STREAM_NEED_FEEDBACK, STREAM_CLOSED, STREAM_HANDED_OVER = 1, 2, 4, 8
STREAM_MSG_IN_INPUT = 1
STREAM_EV_REMOTE_CONSUMED_MOVED, STREAM_EV_CLOSED_BY_RST, STREAM_EV_CLOSED_BY_CLOSE, STREAM_EV_HANDED_OVER, STREAM_EV_WRITABLE = 1, 2, 4, 8, 16
# the sending side (b2_stream_write)
STREAM_WRITE_DT = np.dtype([("stream_id", "<i8"), ("flags", "<u4"), ("src_off", "<u4"), ("src_len", "<u4"), ("reserved", "<u4")])      # == b2_stream_write_desc
STREAM_WRITE_RESULT_DT = np.dtype([("status", "<i4"), ("n_frames", "<u4"), ("out_off", "<u4"), ("out_len", "<u4"), ("produced", "<u8"),
                                   ("host_socket_id", "<u8")])
assert STREAM_WRITE_DT.itemsize == 24 and STREAM_WRITE_RESULT_DT.itemsize == 32
STREAM_W_FROM_MSG = 1
STREAM_W_NOT_CONNECTED, STREAM_W_HANDED_OVER = -1, -2
STREAM_W_DEFAULT_SEGMENT = 512 << 20          # -stream_write_max_segment_size's default (max_segment_size 0)


class Method(C.Structure):
    _fields_ = [("service_full_name", C.c_char_p), ("service_name", C.c_char_p), ("method_name", C.c_char_p),
                ("request_type_name", C.c_char_p), ("handler", C.c_int32), ("echo_attachment", C.c_int32),
                ("response_checksum_type", C.c_int32), ("response_compress_type", C.c_int32)]


class Options(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_batch_bytes", C.c_uint32), ("max_msgs", C.c_uint32),
                ("max_runs", C.c_uint32), ("max_resp_bytes", C.c_uint32), ("tile_bytes", C.c_uint32),
                ("max_body_size", C.c_uint64)]


class BatchResult(C.Structure):
    _fields_ = [("runs", C.c_void_p), ("n_runs", C.c_uint32),
                ("msgs", C.c_void_p), ("n_msgs", C.c_uint32),
                ("resp", C.c_void_p), ("resp_bytes", C.c_uint32),
                ("kernel_ms", C.c_float), ("n_launches", C.c_uint32), ("refs", C.c_void_p), ("iov", C.c_void_p)]


class H2RingResult(C.Structure):
    _fields_ = [("runs", C.c_void_p), ("n_runs", C.c_uint32), ("n_msgs", C.c_uint32), ("msgs", C.c_void_p), ("out", C.c_void_p),
                ("region", C.c_uint32), ("replies", C.c_void_p), ("spans", C.c_void_p), ("status", C.c_int32)]


assert C.sizeof(H2RingResult) == 64


class H2RingTurnResult(C.Structure):
    _fields_ = [("ring", H2RingResult), ("n_resps", C.c_uint32), ("reserved", C.c_uint32), ("resp_offs", C.c_void_p), ("resp_lens", C.c_void_p),
                ("resp_out", C.c_void_p)]


assert C.sizeof(H2RingTurnResult) == 96


class H2ClientRingResult(C.Structure):
    _fields_ = [("runs", C.c_void_p), ("n_runs", C.c_uint32), ("n_calls", C.c_uint32), ("calls", C.c_void_p), ("out", C.c_void_p),
                ("region", C.c_uint32), ("n_reqs", C.c_uint32), ("reqs", C.c_void_p), ("req_out", C.c_void_p), ("status", C.c_int32),
                ("reserved", C.c_uint32)]


assert C.sizeof(H2ClientRingResult) == 64


class ClientRingResult(C.Structure):
    _fields_ = [("batch", BatchResult), ("n_reqs", C.c_uint32), ("reserved", C.c_uint32), ("req_offs", C.c_void_p), ("req_lens", C.c_void_p),
                ("req_out", C.c_void_p)]


assert C.sizeof(ClientRingResult) == 104


class RingTurnResult(C.Structure):
    _fields_ = [("batch", BatchResult), ("n_replies", C.c_uint32), ("reserved", C.c_uint32), ("reply_offs", C.c_void_p), ("reply_lens", C.c_void_p),
                ("reply_out", C.c_void_p)]


assert C.sizeof(RingTurnResult) == 104


class StreamRingResult(C.Structure):
    _fields_ = [("batch", BatchResult), ("n_writes", C.c_uint32), ("out_bytes", C.c_uint32), ("results", C.c_void_p), ("out", C.c_void_p)]


assert C.sizeof(StreamRingResult) == 96


class StreamState(C.Structure):
    _fields_ = [("local_consumed", C.c_uint64), ("remote_consumed", C.c_uint64), ("pending_bytes", C.c_uint32), ("flags", C.c_uint32),
                ("error_code", C.c_int32), ("reserved", C.c_uint32)]


class StreamBatchResult(C.Structure):
    _fields_ = [("msgs", C.c_void_p), ("n_msgs", C.c_uint32), ("events", C.c_void_p), ("n_events", C.c_uint32),
                ("out", C.c_void_p), ("out_bytes", C.c_uint32), ("ctrl", C.c_void_p), ("ctrl_bytes", C.c_uint32),
                ("run_ctrl", C.c_void_p), ("n_runs", C.c_uint32)]


REF_DT = np.dtype([("prefix_len", "<u4"), ("src_off", "<u4"), ("src_len", "<u4"), ("reserved", "<u4")])
IOVEC_DT = np.dtype([("base", "<u8"), ("len", "<u8")])          # struct iovec
INPUT_COPY, INPUT_PULL, RESP_COPY, RESP_BY_REF, RESP_IOVEC = 0, 1, 0, 1, 2


class ResidentKernel(C.Structure):
    _fields_ = [("name", C.c_char_p), ("regs", C.c_uint32), ("threads", C.c_uint32), ("smem_bytes", C.c_uint32), ("fits", C.c_uint32)]


class B2Error(RuntimeError):
    def __init__(self, code, text):
        super().__init__("b2rpc error %d: %s" % (code, text))
        self.code = code


def _load():
    if not os.path.exists(lib_path):
        raise ImportError("brpc_b200/libb2rpc.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a).  There is no CPU fallback.")
    l = C.CDLL(lib_path)
    l.b2_last_error.restype = C.c_char_p
    l.b2_version.restype = C.c_char_p
    l.b2_ctx_create.argtypes = [C.POINTER(Options), C.POINTER(C.c_void_p)]
    l.b2_ctx_destroy.argtypes = [C.c_void_p]
    l.b2_register_method.argtypes = [C.c_void_p, C.POINTER(Method)]
    l.b2_set_server_identity.argtypes = [C.c_void_p, C.c_char_p]
    l.b2_set_stream_handler.argtypes = [C.c_void_p, C.c_int]
    l.b2_set_protocols.argtypes = [C.c_void_p, C.c_uint32]
    l.b2_set_walk_group.argtypes = [C.c_void_p, C.c_uint32]
    l.b2_walk_group.argtypes = [C.c_void_p]
    l.b2_block_alloc.restype = C.c_void_p; l.b2_block_alloc.argtypes = [C.c_size_t]
    l.b2_block_free.argtypes = [C.c_void_p]
    l.b2_block_pool_host_allocs.restype = C.c_uint64
    l.b2_set_modes.argtypes = [C.c_void_p, C.c_int, C.c_int]
    l.b2_ring_start.argtypes = [C.c_void_p]; l.b2_ring_stop.argtypes = [C.c_void_p]
    l.b2_ring_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_ring_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(BatchResult)]
    l.b2_ring_launches.restype = C.c_uint64; l.b2_ring_launches.argtypes = [C.c_void_p]
    l.b2_ring_phase_ns.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    l.b2_latency_probe.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p]
    l.b2_process_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(BatchResult)]
    l.b2_batch_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    l.b2_batch_collect.argtypes = [C.c_void_p, C.POINTER(BatchResult)]
    l.b2_batch_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    l.b2_batch_execute.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_uint32)]
    l.b2_batch_execute_many.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_uint32)]
    l.b2_batch_launch.argtypes = [C.c_void_p]
    l.b2_batch_wait.argtypes = [C.c_void_p]
    l.b2_elapsed_ms.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]
    l.b2_batch_download.argtypes = [C.c_void_p, C.POINTER(BatchResult)]
    l.b2_batch_info.argtypes = [C.c_void_p, C.c_void_p]
    l.b2_resident_plan.argtypes = [C.c_void_p, C.POINTER(ResidentKernel), C.c_int]
    l.b2_device_pci_bus_id.argtypes = [C.c_int, C.c_char_p, C.c_int]
    l.b2_stage_times.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.c_int]
    l.b2_crc32c_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    l.b2_snappy_uncompress_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                             C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    l.b2_snappy_compress_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                           C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    l.b2_crc32c_extend.restype = C.c_uint32; l.b2_crc32c_extend.argtypes = [C.c_uint32, C.c_char_p, C.c_size_t]
    l.b2_snappy_max_compressed_length.restype = C.c_size_t; l.b2_snappy_max_compressed_length.argtypes = [C.c_size_t]
    l.b2_snappy_raw_compress.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t)]
    l.b2_snappy_get_uncompressed_length.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    l.b2_snappy_raw_uncompress.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p]
    l.b2_hpack_reset.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    l.b2_hpack_decode_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                        C.c_void_p, C.c_void_p, C.c_void_p]
    l.b2_h2_scan_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                   C.c_void_p, C.c_void_p, C.c_void_p]
    l.b2_h2_conn_reset.argtypes = [C.c_void_p, C.c_uint32]
    l.b2_h2_configure.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_h2_process_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                      C.POINTER(C.c_uint32), C.c_void_p, C.c_uint32]
    l.b2_h2_pack_requests.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    l.b2_h2_conn_set_next_stream_id.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    l.b2_h2_conn_peer_update.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    l.b2_h2_client_conn_reset.argtypes = [C.c_void_p, C.c_uint32]
    l.b2_h2_client_process_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                             C.POINTER(C.c_uint32), C.c_void_p, C.c_uint32]
    l.b2_h2_client_abandon_streams.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    l.b2_h2_conn_set_gunzip.argtypes = [C.c_void_p, C.c_uint32, C.c_int]
    l.b2_h2_serve_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                    C.POINTER(C.c_uint32), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    l.b2_h2_ring_enable.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_h2_ring_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_h2_ring_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(H2RingResult)]
    l.b2_h2_ring_turn_enable.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_h2_ring_turn_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_h2_ring_turn_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(H2RingTurnResult)]
    l.b2_h2_client_ring_enable.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_h2_client_ring_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_h2_client_ring_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(H2ClientRingResult)]
    l.b2_client_ring_enable.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_client_ring_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_client_ring_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(ClientRingResult)]
    l.b2_ring_turn_enable.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_ring_turn_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_ring_turn_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(RingTurnResult)]
    l.b2_h2_pack_responses.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    l.b2_pack_requests.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    l.b2_pack_responses.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    l.b2_stream_configure.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_stream_open.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    l.b2_stream_set_connected.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_stream_close.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_stream_query.argtypes = [C.c_void_p, C.c_int64, C.POINTER(StreamState)]
    l.b2_stream_take_pending.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_stream_results.argtypes = [C.c_void_p, C.POINTER(StreamBatchResult)]
    l.b2_stream_ring_enable.argtypes = [C.c_void_p, C.c_uint32]
    l.b2_stream_write.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    l.b2_stream_ring_write_enable.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    l.b2_stream_ring_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    l.b2_stream_ring_wait.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(StreamRingResult)]
    l.b2_counters_read.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    l.b2_counters_device_ptr.restype = C.c_void_p; l.b2_counters_device_ptr.argtypes = [C.c_void_p]
    return l


lib = _load()

# every symbol include/b2rpc.h declares (tests check the library exports them)
ABI_SYMBOLS = ["b2_ctx_create", "b2_ctx_destroy", "b2_last_error", "b2_version", "b2_register_method",
               "b2_set_server_identity", "b2_set_stream_handler", "b2_set_protocols", "b2_block_alloc", "b2_block_free", "b2_block_pool_host_allocs", "b2_set_modes", "b2_ring_start", "b2_ring_stop", "b2_ring_submit", "b2_ring_wait", "b2_ring_launches", "b2_ring_phase_ns", "b2_latency_probe", "b2_process_batch", "b2_batch_submit", "b2_batch_collect", "b2_batch_upload",
               "b2_batch_execute", "b2_batch_execute_many", "b2_batch_download", "b2_batch_launch", "b2_batch_wait",
               "b2_elapsed_ms", "b2_batch_info", "b2_set_walk_group", "b2_walk_group", "b2_resident_plan", "b2_device_pci_bus_id", "b2_stage_times", "b2_crc32c_batch", "b2_crc32c_extend", "b2_snappy_max_compressed_length", "b2_snappy_raw_compress", "b2_snappy_get_uncompressed_length", "b2_snappy_raw_uncompress", "b2_snappy_uncompress_batch", "b2_snappy_compress_batch", "b2_hpack_reset", "b2_hpack_decode_batch", "b2_pack_requests", "b2_pack_responses", "b2_h2_scan_batch", "b2_h2_conn_reset", "b2_h2_configure", "b2_h2_process_batch", "b2_h2_pack_responses", "b2_counters_read",
               "b2_counters_device_ptr", "b2_counters_allreduce", "b2_h2_pack_requests", "b2_h2_conn_set_next_stream_id", "b2_h2_conn_peer_update",
               "b2_h2_client_conn_reset", "b2_h2_client_process_batch", "b2_h2_client_abandon_streams", "b2_h2_conn_set_gunzip",
               "b2_h2_serve_batch", "b2_stream_configure", "b2_stream_open", "b2_stream_set_connected", "b2_stream_close", "b2_stream_query",
               "b2_stream_take_pending", "b2_stream_results", "b2_stream_write", "b2_stream_ring_enable", "b2_h2_ring_enable", "b2_h2_ring_submit",
               "b2_h2_ring_wait", "b2_h2_ring_turn_enable", "b2_h2_ring_turn_submit", "b2_h2_ring_turn_wait", "b2_h2_client_ring_enable", "b2_h2_client_ring_submit", "b2_h2_client_ring_wait", "b2_client_ring_enable",
               "b2_client_ring_submit", "b2_client_ring_wait", "b2_ring_turn_enable", "b2_ring_turn_submit", "b2_ring_turn_wait",
               "b2_stream_ring_write_enable", "b2_stream_ring_submit", "b2_stream_ring_wait"]

ECHO_METHOD = dict(service_full_name=b"example.EchoService", service_name=b"EchoService", method_name=b"Echo",
                   request_type_name=b"example.EchoRequest", handler=1, echo_attachment=1,
                   response_checksum_type=0, response_compress_type=0)


def _check(rc):
    if rc < 0:
        raise B2Error(rc, (lib.b2_last_error() or b"").decode("utf-8", "replace"))
    return rc


def _view(ptr, nbytes, dtype=np.uint8):
    """nbytes of context-owned memory at ptr as a dtype array (no copy)"""
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr)).view(dtype) if nbytes else np.zeros(0, dtype)


def _h2_ring_views(res):
    """(run_status, msgs, out, replies, spans) of an H2RingResult: out covers n_runs * region bytes, replies every span"""
    n = res.n_runs
    spans = _view(res.spans, 16 * n, H2_REPLY_SPAN_DT)
    rep_end = int((spans["off"].astype(np.int64) + spans["len"]).max()) if n else 0
    return (_view(res.runs, 32 * n, H2_RUN_STATUS_DT), _view(res.msgs, 64 * res.n_msgs, H2_MSG_DT), _view(res.out, res.region * n),
            _view(res.replies, rep_end), spans)


# The cyclic garbage collector runs at whatever allocation crosses its threshold — inside a latency loop as well — and b2_ctx_destroy waits
# for the whole device, including another context's resident ring kernel until that one idles out (B2_RING_IDLE_MS).  A Context the
# collector reclaims is therefore destroyed at the next safe point instead: the next Context creation or close(), or exit.
_in_gc = [False]
_reclaimed = []


def _gc_phase(phase, info):
    _in_gc[0] = phase == "start"


def _destroy_reclaimed():
    hs = _reclaimed[:]
    del _reclaimed[:]
    for h in hs:
        lib.b2_ring_stop(h)          # every resident kernel among them leaves first: each destroy waits for the device
    for h in hs:
        lib.b2_ctx_destroy(h)


gc.callbacks.append(_gc_phase)
atexit.register(_destroy_reclaimed)


class PinnedBuffer:
    """Host memory from b2_block_alloc (cudaHostAlloc), viewed as a numpy uint8 array."""

    def __init__(self, nbytes):
        self.ptr = lib.b2_block_alloc(nbytes)
        if not self.ptr:
            raise B2Error(B2_E_NOMEM, "b2_block_alloc failed")
        self.nbytes = nbytes
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))

    def free(self):
        if self.ptr:
            lib.b2_block_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    """b2_ctx: one per GPU."""

    def __init__(self, device=0, max_batch_bytes=64 << 20, max_msgs=1 << 20, max_runs=4096, max_resp_bytes=0,
                 tile_bytes=0, max_body_size=0, methods=(ECHO_METHOD,), server_identity=None, stream_handler=0):
        _destroy_reclaimed()
        opt = Options(device, max_batch_bytes, max_msgs, max_runs, max_resp_bytes, tile_bytes, max_body_size)
        h = C.c_void_p()
        _check(lib.b2_ctx_create(C.byref(opt), C.byref(h)))
        self._h = h
        self._keep = []
        for m in methods:
            self.register_method(**m)
        if server_identity:
            _check(lib.b2_set_server_identity(self._h, server_identity))
        if stream_handler:
            _check(lib.b2_set_stream_handler(self._h, stream_handler))

    def close(self):
        if getattr(self, "_h", None):
            lib.b2_ctx_destroy(self._h)
            self._h = None
        _destroy_reclaimed()

    def __del__(self):
        try:
            if _in_gc[0] and getattr(self, "_h", None):
                _reclaimed.append(self._h)
                self._h = None
            else:
                self.close()
        except Exception:
            pass

    def register_method(self, **kw):
        m = Method(**kw)
        self._keep.append(m)
        return _check(lib.b2_register_method(self._h, C.byref(m)))

    @staticmethod
    def _views(res):
        runs = np.ctypeslib.as_array((C.c_uint8 * (32 * res.n_runs)).from_address(res.runs)).view(RUN_STATUS_DT) \
            if res.n_runs else np.zeros(0, RUN_STATUS_DT)
        msgs = np.ctypeslib.as_array((C.c_uint8 * (64 * res.n_msgs)).from_address(res.msgs)).view(MSG_DT) \
            if res.n_msgs else np.zeros(0, MSG_DT)
        resp = np.ctypeslib.as_array((C.c_uint8 * res.resp_bytes).from_address(res.resp)) \
            if res.resp_bytes else np.zeros(0, np.uint8)
        return runs, msgs, resp

    @staticmethod
    def _info(res):
        refs = None
        if res.refs and res.n_msgs:
            refs = np.ctypeslib.as_array((C.c_uint8 * (16 * res.n_msgs)).from_address(res.refs)).view(REF_DT)
        iov = None
        if res.iov and res.n_msgs:
            iov = np.ctypeslib.as_array((C.c_uint8 * (32 * res.n_msgs)).from_address(res.iov)).view(IOVEC_DT)
        return {"kernel_ms": res.kernel_ms, "n_launches": res.n_launches, "refs": refs, "iov": iov}

    # ---- the persistent latency kernel (b2_ring_*) ----
    def _ring_bytes(self, data, ptr, nbytes):
        """a ticket's bytes: (ptr, nbytes) as given, else data's, which the context keeps referenced until the next submission"""
        if ptr is None:
            data = np.ascontiguousarray(data, dtype=np.uint8); ptr, nbytes = data.ctypes.data, data.nbytes
            self._ring_keep = data
        return ptr, nbytes

    def ring_start(self):
        _check(lib.b2_ring_start(self._h))

    def ring_stop(self):
        _check(lib.b2_ring_stop(self._h))

    def ring_submit(self, data, runs, ptr=None, nbytes=None):
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        ptr, nbytes = self._ring_bytes(data, ptr, nbytes)
        t = C.c_uint32(0)
        _check(lib.b2_ring_submit(self._h, ptr, nbytes, runs.ctypes.data, len(runs), C.byref(t)))
        return t.value

    def ring_wait(self, ticket):
        res = BatchResult()
        _check(lib.b2_ring_wait(self._h, ticket, C.byref(res)))
        rs, msgs, resp = self._views(res)
        return rs, msgs, resp, self._info(res)

    def latency_probe(self, ptr, nbytes, runs, iters, use_ring):
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        us = np.zeros(iters, np.float32)
        _check(lib.b2_latency_probe(self._h, ptr, nbytes, runs.ctypes.data, len(runs), iters, 1 if use_ring else 0, us.ctypes.data))
        return us

    def ring_phase_ns(self, ticket):
        out = (C.c_uint64 * 4)()
        _check(lib.b2_ring_phase_ns(self._h, ticket, out))
        return list(out)

    def ring_launches(self):
        return int(lib.b2_ring_launches(self._h))

    def set_protocols(self, mask):
        _check(lib.b2_set_protocols(self._h, mask))

    def set_walk_group(self, mode):
        """Tiles per walk group of the front stages: 0 auto, 1 one tile per group, 2..8 forced (b2_set_walk_group); upload again after."""
        _check(lib.b2_set_walk_group(self._h, mode))

    def walk_group(self):
        """The walk group size the last launch used."""
        return _check(lib.b2_walk_group(self._h))

    def set_modes(self, input_mode=INPUT_COPY, resp_mode=RESP_COPY):
        _check(lib.b2_set_modes(self._h, input_mode, resp_mode))

    def process_batch(self, data, runs):
        """Host buffers in, host (pinned) views out: (run_status, msgs, resp, info)."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        res = BatchResult()
        _check(lib.b2_process_batch(self._h, data.ctypes.data, data.nbytes, runs.ctypes.data, len(runs), C.byref(res)))
        rs, msgs, resp = self._views(res)
        return rs, msgs, resp, self._info(res)

    def upload(self, data, runs):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        _check(lib.b2_batch_upload(self._h, data.ctypes.data, data.nbytes, runs.ctypes.data, len(runs)))

    def upload_ptr(self, ptr, nbytes, runs):
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        _check(lib.b2_batch_upload(self._h, ptr, nbytes, runs.ctypes.data, len(runs)))

    def execute(self):
        ms, n = C.c_float(0), C.c_uint32(0)
        _check(lib.b2_batch_execute(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def execute_many(self, steps):
        ms, n = C.c_float(0), C.c_uint32(0)
        _check(lib.b2_batch_execute_many(self._h, steps, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def launch(self):
        _check(lib.b2_batch_launch(self._h))

    def wait(self):
        _check(lib.b2_batch_wait(self._h))

    def elapsed_ms_to(self, other):
        ms = C.c_float(0)
        _check(lib.b2_elapsed_ms(self._h, other._h, C.byref(ms)))
        return ms.value

    def download(self):
        res = BatchResult()
        _check(lib.b2_batch_download(self._h, C.byref(res)))
        rs, msgs, resp = self._views(res)
        return rs, msgs, resp, self._info(res)

    def process_batch_ptr(self, ptr, nbytes, runs):
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        res = BatchResult()
        _check(lib.b2_process_batch(self._h, ptr, nbytes, runs.ctypes.data, len(runs), C.byref(res)))
        rs, msgs, resp = self._views(res)
        return rs, msgs, resp, self._info(res)

    def submit_ptr(self, ptr, nbytes, runs):
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        self._submitted_runs = runs           # keep alive until collect
        _check(lib.b2_batch_submit(self._h, ptr, nbytes, runs.ctypes.data, len(runs)))

    def collect(self):
        res = BatchResult()
        _check(lib.b2_batch_collect(self._h, C.byref(res)))
        rs, msgs, resp = self._views(res)
        return rs, msgs, resp, self._info(res)

    # ---- the stream table: the receiving side of brpc's Stream on the device (b2_stream_*) ----
    def stream_configure(self, max_streams, pending_bytes, out_bytes=0):
        _check(lib.b2_stream_configure(self._h, max_streams, pending_bytes, out_bytes))

    def stream_open(self, streams):
        """streams: STREAM_DESC_DT array or a list of (stream_id, remote_stream_id, host_socket_id, flags[, max_buf_size])."""
        if not isinstance(streams, np.ndarray):
            a = np.zeros(len(streams), STREAM_DESC_DT)
            for i, t in enumerate(streams):
                a[i] = tuple(t) + (0,) * (5 - len(t))
            streams = a
        streams = np.ascontiguousarray(streams, dtype=STREAM_DESC_DT)
        _check(lib.b2_stream_open(self._h, streams.ctypes.data, len(streams)))

    def stream_set_connected(self, stream_id, remote_stream_id, flags=0):
        """Returns the FEEDBACK frame SetConnected writes (b"" = none)."""
        buf = C.create_string_buffer(64); n = C.c_uint32(0)
        _check(lib.b2_stream_set_connected(self._h, stream_id, remote_stream_id, flags, buf, 64, C.byref(n)))
        return buf.raw[:n.value]

    def stream_close(self, stream_id):
        """Returns the CLOSE frame to write (b"" = none)."""
        buf = C.create_string_buffer(64); n = C.c_uint32(0)
        _check(lib.b2_stream_close(self._h, stream_id, buf, 64, C.byref(n)))
        return buf.raw[:n.value]

    def stream_query(self, stream_id):
        st = StreamState()
        _check(lib.b2_stream_query(self._h, stream_id, C.byref(st)))
        return {"local_consumed": st.local_consumed, "remote_consumed": st.remote_consumed, "pending_bytes": st.pending_bytes,
                "flags": st.flags, "error_code": st.error_code}

    def stream_take_pending(self, stream_id, cap):
        buf = np.zeros(max(1, cap), np.uint8); n = C.c_uint32(0)
        _check(lib.b2_stream_take_pending(self._h, stream_id, buf.ctypes.data, cap, C.byref(n)))
        return buf[:n.value].tobytes()

    def stream_ring_enable(self, out_bytes):
        """Run the stream pass on the ring too (b2_stream_ring_enable): after stream_configure, before the first ring call."""
        _check(lib.b2_stream_ring_enable(self._h, out_bytes))

    def stream_results(self):
        """(msgs, events, out, ctrl, run_ctrl) of the last collected batch or ring ticket: views of context-owned memory, valid until the
        next batch call (a ring ticket's: until its slot is reused)."""
        r = StreamBatchResult()
        _check(lib.b2_stream_results(self._h, C.byref(r)))
        return (_view(r.msgs, 32 * r.n_msgs, STREAM_MSG_DT), _view(r.events, 80 * r.n_events, STREAM_EVENT_DT), _view(r.out, r.out_bytes, np.uint8),
                _view(r.ctrl, r.ctrl_bytes, np.uint8), _view(r.run_ctrl, 8 * r.n_runs, np.uint32).reshape(-1, 2))

    @staticmethod
    def _write_list(writes):
        """STREAM_WRITE_DT array of writes given as such an array or as a list of (stream_id, flags, src_off, src_len)"""
        if not isinstance(writes, np.ndarray):
            a = np.zeros(len(writes), STREAM_WRITE_DT)
            for i, t in enumerate(writes):
                a[i] = tuple(t) + (0,) * (5 - len(t))
            writes = a
        return np.ascontiguousarray(writes, dtype=STREAM_WRITE_DT)

    def stream_write(self, writes, data=None, max_segment_size=0, out_cap=None, out=None):
        """StreamWrite for a batch of writes (b2_stream_write).  writes: STREAM_WRITE_DT array or a list of (stream_id, flags, src_off,
        src_len); data: the bytes host-sourced writes index.  Returns (results, out): write i's frames are
        out[results[i]["out_off"]:results[i]["out_off"] + results[i]["out_len"]]."""
        writes = self._write_list(writes)
        n = len(writes)
        if data is None:
            ptr, nb = None, 0
        else:
            data = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
            ptr, nb = data.ctypes.data, data.nbytes
        if out is None:
            if out_cap is None:         # the bound the call checks: align16(len + ceil(len / seg) * 38) per write
                seg = max_segment_size or STREAM_W_DEFAULT_SEGMENT
                lens = np.where(writes["flags"] & STREAM_W_FROM_MSG, 0, writes["src_len"]).astype(np.int64)
                if np.any(writes["flags"] & STREAM_W_FROM_MSG):
                    sm = self.stream_results()[0]
                    fm = (writes["flags"] & STREAM_W_FROM_MSG) != 0
                    idx = writes["src_off"][fm].astype(np.int64)
                    lens[fm] = np.where(idx < len(sm), sm["len"][np.minimum(idx, max(len(sm) - 1, 0))] if len(sm) else 0, 0)
                nfr = np.maximum(1, (lens + seg - 1) // seg)
                out_cap = int(((lens + nfr * 38 + 15) // 16 * 16).sum())
            out = np.empty(max(1, out_cap), np.uint8)
        res = np.zeros(n, STREAM_WRITE_RESULT_DT)
        _check(lib.b2_stream_write(self._h, ptr, nb, writes.ctypes.data, n, max_segment_size, out.ctypes.data, out.nbytes, res.ctypes.data))
        return res, out

    def batch_info(self):
        out = (C.c_uint32 * 4)()
        _check(lib.b2_batch_info(self._h, out))
        return {"tile_bytes": out[0], "n_tiles": out[1], "spec_k": out[2], "fused": bool(out[3])}

    def resident_plan(self):
        """k_fused in the uploaded batch's shape, then the kernels launched between two k_fused passes: registers, threads and shared
        memory per block, and how many blocks of each start on an SM beside one k_fused CTA (b2_resident_plan)."""
        out = (ResidentKernel * 8)()
        n = _check(lib.b2_resident_plan(self._h, out, 8))
        return [{"name": out[i].name.decode(), "regs": out[i].regs, "threads": out[i].threads, "smem_bytes": out[i].smem_bytes,
                 "fits": out[i].fits} for i in range(min(n, 8))]

    def stage_times(self):
        names = (C.c_char_p * 16)()
        ms = (C.c_float * 16)()
        n = lib.b2_stage_times(self._h, names, ms, 16)
        return [(names[i].decode(), ms[i]) for i in range(max(0, min(n, 16)))]

    def crc32c_batch(self, data, offs, lens):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint32)
        lens = np.ascontiguousarray(lens, dtype=np.uint32)
        out = np.zeros(len(offs), dtype=np.uint32)
        _check(lib.b2_crc32c_batch(self._h, data.ctypes.data, data.nbytes, offs.ctypes.data, lens.ctypes.data,
                                   len(offs), out.ctypes.data))
        return out

    def snappy_uncompress_batch(self, data, offs, lens, out_cap):
        """Returns (list of bytes or None) for each slice."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint32); lens = np.ascontiguousarray(lens, dtype=np.uint32)
        n = len(offs)
        out = np.zeros(out_cap, dtype=np.uint8); ooffs = np.zeros(n, dtype=np.uint32); olens = np.zeros(n, dtype=np.int32)
        _check(lib.b2_snappy_uncompress_batch(self._h, data.ctypes.data, data.nbytes, offs.ctypes.data, lens.ctypes.data, n,
                                              out.ctypes.data, out_cap, ooffs.ctypes.data, olens.ctypes.data))
        return [None if olens[i] < 0 else out[ooffs[i]:ooffs[i] + olens[i]].tobytes() for i in range(n)]

    def snappy_compress_batch(self, data, offs, lens, out_cap):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint32); lens = np.ascontiguousarray(lens, dtype=np.uint32)
        n = len(offs)
        out = np.zeros(out_cap, dtype=np.uint8); ooffs = np.zeros(n, dtype=np.uint32); olens = np.zeros(n, dtype=np.uint32)
        _check(lib.b2_snappy_compress_batch(self._h, data.ctypes.data, data.nbytes, offs.ctypes.data, lens.ctypes.data, n,
                                            out.ctypes.data, out_cap, ooffs.ctypes.data, olens.ctypes.data))
        return [out[ooffs[i]:ooffs[i] + olens[i]].tobytes() for i in range(n)]

    def hpack_reset(self, conn, max_table_size=4096):
        _check(lib.b2_hpack_reset(self._h, conn, max_table_size))

    def hpack_decode_batch(self, data, blocks, per_block_cap=4096):
        """blocks: list of (conn, offset, length).  Returns [(status, [(name, value), ...]), ...]."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        b = np.zeros(len(blocks), HPACK_BLOCK_DT)
        for i, (c, o, n) in enumerate(blocks):
            b[i] = (c, o, n, 0)
        n = len(blocks)
        out = np.zeros(max(1, n * per_block_cap), np.uint8); ol = np.zeros(n, np.uint32); st = np.zeros(n, np.int32); nh = np.zeros(n, np.uint32)
        _check(lib.b2_hpack_decode_batch(self._h, data.ctypes.data, data.nbytes, b.ctypes.data, n, out.ctypes.data, per_block_cap,
                                         ol.ctypes.data, st.ctypes.data, nh.ctypes.data))
        res = []
        for i in range(n):
            buf = out[i * per_block_cap:i * per_block_cap + ol[i]]; o = 0; hs = []
            while o < len(buf):
                nl = int(buf[o]) | (int(buf[o + 1]) << 8); vl = int(buf[o + 2]) | (int(buf[o + 3]) << 8)
                hs.append((buf[o + 4:o + 4 + nl].tobytes(), buf[o + 4 + nl:o + 4 + nl + vl].tobytes())); o += 4 + nl + vl
            assert len(hs) == nh[i]
            res.append((int(st[i]), hs))
        return res

    def h2_scan_batch(self, data, runs, max_frame_size=16384, cap_per_run=256):
        data = np.ascontiguousarray(data, dtype=np.uint8); runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        n = len(runs)
        frames = np.zeros(max(1, n * cap_per_run), H2_FRAME_DT); nf = np.zeros(n, np.uint32); cons = np.zeros(n, np.uint32); err = np.zeros(n, np.uint32)
        _check(lib.b2_h2_scan_batch(self._h, data.ctypes.data, data.nbytes, runs.ctypes.data, n, max_frame_size, frames.ctypes.data, cap_per_run,
                                    nf.ctypes.data, cons.ctypes.data, err.ctypes.data))
        return [frames[i * cap_per_run:i * cap_per_run + min(int(nf[i]), cap_per_run)] for i in range(n)], nf, cons, err

    def h2_configure(self, max_conns=1024, max_pending=8, stream_bytes=69632):
        _check(lib.b2_h2_configure(self._h, max_conns, max_pending, stream_bytes))

    def h2_conn_reset(self, conn):
        _check(lib.b2_h2_conn_reset(self._h, conn))

    def h2_process_batch(self, data, runs, msg_cap=None, out_cap=None, out=None):
        """runs[i].socket_id = h2 connection index.  Returns (run_status, msgs, out)."""
        data = np.ascontiguousarray(data, dtype=np.uint8); runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        n = len(runs)
        msg_cap = msg_cap or max(64, 64 * n)
        out_cap = out_cap or max(1 << 16, n * (1 << 17))
        rs = np.zeros(n, H2_RUN_STATUS_DT); msgs = np.zeros(msg_cap, H2_MSG_DT); nm = C.c_uint32(0)
        if out is None:
            out = np.empty(out_cap, np.uint8)       # (pass a PinnedBuffer's array to keep the copies off pageable memory)
        out_cap = out.nbytes
        _check(lib.b2_h2_process_batch(self._h, data.ctypes.data, data.nbytes, runs.ctypes.data, n, rs.ctypes.data, msgs.ctypes.data, msg_cap,
                                       C.byref(nm), out.ctypes.data, out_cap))
        return rs, msgs[:nm.value], out

    def h2_pack_responses(self, data, resps, out_cap=None, raw=False, out=None):
        """resps: H2_RESPONSE_DT array (offsets into data).  Returns the packed bytes of every response."""
        resps = np.ascontiguousarray(resps, dtype=H2_RESPONSE_DT)
        n = len(resps)
        out_cap = out_cap or int(resps["body_len"].astype(np.int64).sum() * 2 + n * 2048 + 4096)
        offs = np.zeros(n, np.uint32); lens = np.zeros(n, np.uint32)
        if out is None:
            out = np.empty(out_cap, np.uint8)
        out_cap = out.nbytes
        if data is None:                 # every field uses a zero-copy source (B2_H2_RESP_*_IN_INPUT / _IN_OUT)
            ptr, nb = None, 0
        else:
            data = np.ascontiguousarray(data, dtype=np.uint8); ptr, nb = data.ctypes.data, data.nbytes
        _check(lib.b2_h2_pack_responses(self._h, ptr, nb, resps.ctypes.data, n, out.ctypes.data, out_cap, offs.ctypes.data, lens.ctypes.data))
        if raw:
            return out, offs, lens
        return [out[offs[i]:offs[i] + lens[i]].tobytes() for i in range(n)]

    def h2_pack_requests(self, data, reqs, out_cap=None):
        """Client side of h2 (H2UnsentRequest): reqs is an H2_REQUEST_DT array (offsets into data).  Returns (results, [bytes per request])."""
        data = np.ascontiguousarray(data, dtype=np.uint8); reqs = np.ascontiguousarray(reqs, dtype=H2_REQUEST_DT)
        n = len(reqs)
        out_cap = out_cap or int(reqs["body_len"].astype(np.int64).sum() * 2 + n * 8192 + 4096)
        res = np.zeros(n, H2_REQUEST_RESULT_DT); out = np.empty(out_cap, np.uint8)
        _check(lib.b2_h2_pack_requests(self._h, data.ctypes.data, data.nbytes, reqs.ctypes.data, n, out.ctypes.data, out_cap, res.ctypes.data))
        return res, [out[r["out_off"]:r["out_off"] + r["out_len"]].tobytes() for r in res]

    def h2_conn_peer_update(self, conn, header_table_size=None, max_frame_size=None, stream_window_size=None, conn_window_add=None):
        """The peer's SETTINGS / connection WINDOW_UPDATE, parsed by the host, mirrored into the device's connection state."""
        u = np.zeros(1, H2_PEER_UPDATE_DT)
        vals = (header_table_size, max_frame_size, stream_window_size, conn_window_add)
        u[0] = (sum(1 << i for i, v in enumerate(vals) if v is not None), *(0 if v is None else v for v in vals))
        _check(lib.b2_h2_conn_peer_update(self._h, conn, u.ctypes.data))

    def h2_conn_set_next_stream_id(self, conn, next_id):
        _check(lib.b2_h2_conn_set_next_stream_id(self._h, conn, next_id))

    def h2_client_conn_reset(self, conn):
        """A new client connection whose server frames the device parses (h2_client_process_batch)."""
        _check(lib.b2_h2_client_conn_reset(self._h, conn))

    def h2_client_process_batch(self, data, runs, call_cap=None, out_cap=None, out=None):
        """The server's bytes of client connections (runs[i].socket_id = connection).  Returns (run_status, calls, out): one H2_CALL_DT per
        stream that left its connection; header records, copied bodies and error texts live in out, the bytes to write back at ctrl_off."""
        data = np.ascontiguousarray(data, dtype=np.uint8); runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        n = len(runs)
        call_cap = call_cap or max(64, 128 * n)
        out_cap = out_cap or max(1 << 16, n * (1 << 17))
        rs = np.zeros(n, H2_RUN_STATUS_DT); calls = np.zeros(call_cap, H2_CALL_DT); nc = C.c_uint32(0)
        if out is None:
            out = np.empty(out_cap, np.uint8)
        out_cap = out.nbytes
        _check(lib.b2_h2_client_process_batch(self._h, data.ctypes.data, data.nbytes, runs.ctypes.data, n, rs.ctypes.data, calls.ctypes.data,
                                              call_cap, C.byref(nc), out.ctypes.data, out_cap))
        return rs, calls[:nc.value], out

    def h2_client_abandon_streams(self, conn, stream_ids):
        """Calls given up on (AddAbandonedStream): their streams are dropped at the end of the connection's next client parse."""
        ids = np.ascontiguousarray(stream_ids, dtype=np.uint32)
        _check(lib.b2_h2_client_abandon_streams(self._h, conn, ids.ctypes.data, len(ids)))

    def h2_conn_set_gunzip(self, conn, enable=True):
        """The connection's gzip-compressed messages are inflated on the device by the next batches (H2_FLAG_GUNZIPPED: msg_off / msg_len
        then index the inflated bytes in out; H2_FLAG_GUNZIP_HOST: left for the host).  h2_conn_reset / h2_client_conn_reset clear it."""
        _check(lib.b2_h2_conn_set_gunzip(self._h, conn, 1 if enable else 0))

    def h2_serve_batch(self, data, runs, msg_cap=None, out_cap=None, replies_cap=None, out=None, replies=None):
        """h2_process_batch that also answers the gRPC calls of device echo methods (b2_h2_serve_batch).  Returns (run_status, msgs, out,
        replies, spans): answered calls carry H2_FLAG_ANSWERED and their grpc-status in msgs["reserved"]; run i's replies are
        replies[spans[i]["off"]:spans[i]["off"] + spans[i]["len"]], to be written after its control bytes."""
        data = np.ascontiguousarray(data, dtype=np.uint8); runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        n = len(runs)
        msg_cap = msg_cap or max(64, 64 * n)
        out_cap = out_cap or max(1 << 16, n * (1 << 17))
        replies_cap = replies_cap or max(1 << 16, n * (1 << 17))
        rs = np.zeros(n, H2_RUN_STATUS_DT); msgs = np.zeros(msg_cap, H2_MSG_DT); nm = C.c_uint32(0); spans = np.zeros(n, H2_REPLY_SPAN_DT)
        if out is None:
            out = np.empty(out_cap, np.uint8)
        if replies is None:
            replies = np.empty(replies_cap, np.uint8)
        _check(lib.b2_h2_serve_batch(self._h, data.ctypes.data, data.nbytes, runs.ctypes.data, n, rs.ctypes.data, msgs.ctypes.data, msg_cap,
                                     C.byref(nm), out.ctypes.data, out.nbytes, replies.ctypes.data, replies.nbytes, spans.ctypes.data))
        return rs, msgs[:nm.value], out, replies, spans

    # ---- h2/gRPC on the latency path (b2_h2_ring_*) ----
    def h2_ring_enable(self, max_bytes, msg_cap, out_cap, replies_cap):
        """Serve h2 batches on the resident k_h2_ring with these per-ticket caps (b2_h2_ring_enable): after h2_configure, before the first
        ring call."""
        _check(lib.b2_h2_ring_enable(self._h, max_bytes, msg_cap, out_cap, replies_cap))

    def h2_ring_submit(self, data, runs, ptr=None, nbytes=None):
        """One batch of server connection runs (runs[i].socket_id = connection).  Returns the ticket."""
        runs = np.ascontiguousarray(runs, dtype=RUN_DT)
        ptr, nbytes = self._ring_bytes(data, ptr, nbytes)
        t = C.c_uint32(0)
        _check(lib.b2_h2_ring_submit(self._h, ptr, nbytes, runs.ctypes.data, len(runs), C.byref(t)))
        return t.value

    def h2_ring_wait(self, ticket):
        """(run_status, msgs, out, replies, spans) of the ticket, as h2_serve_batch returns them: views of the ticket's pinned slot, valid
        until the slot is reused by the 8th later submission.  out covers n_runs * region bytes, replies every span."""
        res = H2RingResult()
        _check(lib.b2_h2_ring_wait(self._h, ticket, C.byref(res)))
        if res.status < 0:
            raise B2Error(res.status, "h2 ring ticket %d" % ticket)
        return _h2_ring_views(res)

    def h2_ring_turn_enable(self, max_bytes, msg_cap, out_cap, replies_cap, max_resps, resp_out_cap):
        """h2_ring_enable whose tickets may also carry the replies the host produced (b2_h2_ring_turn_enable): at most max_resps of them,
        framed within resp_out_cap bytes, per turn."""
        _check(lib.b2_h2_ring_turn_enable(self._h, max_bytes, msg_cap, out_cap, replies_cap, max_resps, resp_out_cap))

    def h2_ring_turn_submit(self, data, runs, resps, ptr=None, nbytes=None):
        """One turn of a gRPC server's event loop: the runs are served as by h2_serve_batch, then resps (H2_RESPONSE_DT, offsets into the
        same data, no zero-copy flags) are packed as by h2_pack_responses.  Either list may be empty, not both.  Returns the ticket."""
        runs = np.ascontiguousarray(runs, dtype=RUN_DT); resps = np.ascontiguousarray(resps, dtype=H2_RESPONSE_DT)
        ptr, nbytes = self._ring_bytes(data, ptr, nbytes)
        t = C.c_uint32(0)
        _check(lib.b2_h2_ring_turn_submit(self._h, ptr, nbytes, runs.ctypes.data if len(runs) else None, len(runs),
                                          resps.ctypes.data if len(resps) else None, len(resps), C.byref(t)))
        return t.value

    def h2_ring_turn_wait(self, ticket):
        """(status, served, [frames per host reply]): status is what h2_serve_batch would have returned for the runs (0, or B2_E_CAPACITY,
        when served lists no messages); served is (run_status, msgs, out, replies, spans) as h2_ring_wait returns them (views of the slot);
        the frames are copies."""
        res = H2RingTurnResult()
        _check(lib.b2_h2_ring_turn_wait(self._h, ticket, C.byref(res)))
        n = res.n_resps
        offs, lens = _view(res.resp_offs, 4 * n, np.uint32), _view(res.resp_lens, 4 * n, np.uint32)
        end = int((offs.astype(np.int64) + lens).max()) if n else 0
        frames = _view(res.resp_out, end)
        return res.ring.status, _h2_ring_views(res.ring), [frames[int(o):int(o) + int(ln)].tobytes() for o, ln in zip(offs, lens)]

    # ---- h2/gRPC client connections on the latency path (b2_h2_client_ring_*) ----
    def h2_client_ring_enable(self, max_bytes, call_cap, out_cap, max_reqs, req_out_cap):
        """Run client connections on the resident k_h2_client_ring with these per-ticket caps (b2_h2_client_ring_enable): after
        h2_configure, before the first ring call."""
        _check(lib.b2_h2_client_ring_enable(self._h, max_bytes, call_cap, out_cap, max_reqs, req_out_cap))

    def h2_client_ring_submit(self, data, runs, reqs, ptr=None, nbytes=None):
        """One turn of a client's event loop: the server's bytes of client connections (runs[i].socket_id = connection) are parsed as by
        h2_client_process_batch, then reqs (H2_REQUEST_DT, offsets into the same data) are packed as by h2_pack_requests.  Either list may
        be empty, not both.  Returns the ticket."""
        runs = np.ascontiguousarray(runs, dtype=RUN_DT); reqs = np.ascontiguousarray(reqs, dtype=H2_REQUEST_DT)
        ptr, nbytes = self._ring_bytes(data, ptr, nbytes)
        t = C.c_uint32(0)
        _check(lib.b2_h2_client_ring_submit(self._h, ptr, nbytes, runs.ctypes.data if len(runs) else None, len(runs),
                                            reqs.ctypes.data if len(reqs) else None, len(reqs), C.byref(t)))
        return t.value

    def h2_client_ring_wait(self, ticket):
        """(run_status, calls, out, req_results, [frames per request]) of the ticket, as h2_client_process_batch and h2_pack_requests return
        them: views of the ticket's pinned slot, valid until the slot is reused by the 8th later submission (the frames are copies)."""
        res = H2ClientRingResult()
        _check(lib.b2_h2_client_ring_wait(self._h, ticket, C.byref(res)))
        if res.status < 0:
            raise B2Error(res.status, "h2 client ring ticket %d" % ticket)
        reqs = _view(res.reqs, 16 * res.n_reqs, H2_REQUEST_RESULT_DT)
        end = int((reqs["out_off"].astype(np.int64) + reqs["out_len"]).max()) if res.n_reqs else 0
        frames = _view(res.req_out, end)
        return (_view(res.runs, 32 * res.n_runs, H2_RUN_STATUS_DT), _view(res.calls, 64 * res.n_calls, H2_CALL_DT), _view(res.out, res.region * res.n_runs),
                reqs, [frames[int(r["out_off"]):int(r["out_off"]) + int(r["out_len"])].tobytes() for r in reqs])

    # ---- baidu_std client connections on the latency path (b2_client_ring_*) ----
    def client_ring_enable(self, max_bytes, max_reqs, req_out_cap):
        """Serve client turns on the resident k_ring<RingBody::requests> with these per-ticket caps (b2_client_ring_enable): before the first ring call."""
        _check(lib.b2_client_ring_enable(self._h, max_bytes, max_reqs, req_out_cap))

    def client_ring_submit(self, data, runs, reqs, ptr=None, nbytes=None):
        """One turn of a client's event loop: runs (RUN_DT, the bytes read from client sockets) are served as by ring_submit, then reqs
        (REQUEST_DT, offsets into the same data) are packed as by pack_requests.  Either list may be empty, not both.  Returns the ticket."""
        runs = np.ascontiguousarray(runs, dtype=RUN_DT); reqs = np.ascontiguousarray(reqs, dtype=REQUEST_DT)
        ptr, nbytes = self._ring_bytes(data, ptr, nbytes)
        t = C.c_uint32(0)
        _check(lib.b2_client_ring_submit(self._h, ptr, nbytes, runs.ctypes.data if len(runs) else None, len(runs),
                                         reqs.ctypes.data if len(reqs) else None, len(reqs), C.byref(t)))
        return t.value

    def client_ring_wait(self, ticket):
        """ring_wait's (run_status, msgs, resp, info) of the ticket's runs, then the frame of every request (b"" where it could not be
        packed, as pack_requests returns them).  The first three are views of the ticket's pinned slot, valid until the 8th later
        submission; the frames are copies."""
        res = ClientRingResult()
        _check(lib.b2_client_ring_wait(self._h, ticket, C.byref(res)))
        rs, msgs, resp = self._views(res.batch)
        offs, lens = _view(res.req_offs, 4 * res.n_reqs, np.uint32), _view(res.req_lens, 4 * res.n_reqs, np.uint32)
        frames = [C.string_at(res.req_out + int(o), int(n)) if n else b"" for o, n in zip(offs, lens)]
        return rs, msgs, resp, self._info(res.batch), frames

    # ---- baidu_std server turns on the latency path (b2_ring_turn_*) ----
    def ring_turn_enable(self, max_bytes, max_resps, resp_out_cap):
        """Serve server turns on the resident k_ring<RingBody::replies> with these per-turn caps (b2_ring_turn_enable): before the first ring call."""
        _check(lib.b2_ring_turn_enable(self._h, max_bytes, max_resps, resp_out_cap))

    def ring_turn_submit(self, data, runs, replies, ptr=None, nbytes=None):
        """One turn of a server's event loop: runs (RUN_DT) are served as by ring_submit, then replies (REPLY_DT, the replies the host
        produced, offsets into the same data) are packed as by pack_responses.  Either list may be empty, not both.  Returns the ticket."""
        runs = np.ascontiguousarray(runs, dtype=RUN_DT); replies = np.ascontiguousarray(replies, dtype=REPLY_DT)
        ptr, nbytes = self._ring_bytes(data, ptr, nbytes)
        t = C.c_uint32(0)
        _check(lib.b2_ring_turn_submit(self._h, ptr, nbytes, runs.ctypes.data if len(runs) else None, len(runs),
                                       replies.ctypes.data if len(replies) else None, len(replies), C.byref(t)))
        return t.value

    def ring_turn_wait(self, ticket):
        """ring_wait's (run_status, msgs, resp, info) of the turn's runs, then the frame of every reply (b"" where it was not packed, as
        pack_responses returns them).  The first three are views of the ticket's pinned slot, valid until the 8th later submission; the
        frames are copies."""
        res = RingTurnResult()
        _check(lib.b2_ring_turn_wait(self._h, ticket, C.byref(res)))
        rs, msgs, resp = self._views(res.batch)
        offs, lens = _view(res.reply_offs, 4 * res.n_replies, np.uint32), _view(res.reply_lens, 4 * res.n_replies, np.uint32)
        frames = [C.string_at(res.reply_out + int(o), int(n)) if n else b"" for o, n in zip(offs, lens)]
        return rs, msgs, resp, self._info(res.batch), frames

    # ---- a Stream producer's turn on the latency path (b2_stream_ring_*) ----
    def stream_ring_write_enable(self, max_bytes, max_writes, write_out_cap, max_segment_size=0):
        """Serve producer turns on the resident k_ring with these per-ticket caps (b2_stream_ring_write_enable): after stream_ring_enable,
        before the first ring call."""
        _check(lib.b2_stream_ring_write_enable(self._h, max_bytes, max_writes, write_out_cap, max_segment_size))

    def stream_ring_submit(self, data, runs, writes, ptr=None, nbytes=None):
        """One producer turn: runs (RUN_DT) are served as by ring_submit on a stream ring, then writes (as for stream_write, offsets into
        the same data) are applied as by stream_write.  Either list may be empty, not both.  Returns the ticket; the context keeps data
        referenced until the ticket's slot is reused."""
        runs = np.ascontiguousarray(runs, dtype=RUN_DT); writes = self._write_list(writes)
        own = ptr is None
        ptr, nbytes = self._ring_bytes(data, ptr, nbytes)
        t = C.c_uint32(0)
        _check(lib.b2_stream_ring_submit(self._h, ptr, nbytes, runs.ctypes.data if len(runs) else None, len(runs),
                                         writes.ctypes.data if len(writes) else None, len(writes), C.byref(t)))
        keep = self.__dict__.setdefault("_stream_ring_keep", [None] * 8)
        keep[t.value % 8] = self._ring_keep if own else None      # (an overflowing ticket's wait reads its bytes again)
        return t.value

    def stream_ring_wait(self, ticket):
        """ring_wait's (run_status, msgs, resp, info) of the ticket's runs, then the write results (STREAM_WRITE_RESULT_DT) and the frames
        (write i's at out[out_off:out_off + out_len], the zero gaps included): views of the ticket's pinned slot, valid until the 8th later
        submission."""
        res = StreamRingResult()
        _check(lib.b2_stream_ring_wait(self._h, ticket, C.byref(res)))
        rs, msgs, resp = self._views(res.batch)
        return (rs, msgs, resp, self._info(res.batch), _view(res.results, 32 * res.n_writes, STREAM_WRITE_RESULT_DT),
                _view(res.out, res.out_bytes))

    def pack_requests(self, data, reqs, out_cap=None):
        """reqs: REQUEST_DT array (offsets into data).  Returns the packed frame of every request (b"" = rejected)."""
        data = np.ascontiguousarray(data, dtype=np.uint8); reqs = np.ascontiguousarray(reqs, dtype=REQUEST_DT)
        n = len(reqs)
        out_cap = out_cap or int((reqs["payload_len"].astype(np.int64) * 7 // 6 + reqs["attachment_len"] + 640).sum() + 4096)
        out = np.empty(out_cap, np.uint8); offs = np.zeros(n, np.uint32); lens = np.zeros(n, np.uint32)
        _check(lib.b2_pack_requests(self._h, data.ctypes.data, data.nbytes, reqs.ctypes.data, n, out.ctypes.data, out_cap, offs.ctypes.data, lens.ctypes.data))
        return [out[offs[i]:offs[i] + lens[i]].tobytes() for i in range(n)]

    def pack_responses(self, data, replies, out_cap=None):
        """replies: REPLY_DT array (offsets into data).  Returns the frame of every reply (b"" = not packable)."""
        data = np.ascontiguousarray(data, dtype=np.uint8); replies = np.ascontiguousarray(replies, dtype=REPLY_DT)
        n = len(replies)
        out_cap = out_cap or int((replies["body_len"].astype(np.int64) * 7 // 6 + replies["attachment_len"] + replies["error_text_len"] + 1024).sum() + data.nbytes + 4096)
        out = np.empty(out_cap, np.uint8); offs = np.zeros(n, np.uint32); lens = np.zeros(n, np.uint32)
        _check(lib.b2_pack_responses(self._h, data.ctypes.data, data.nbytes, replies.ctypes.data, n, out.ctypes.data, out_cap, offs.ctypes.data, lens.ctypes.data))
        return [out[offs[i]:offs[i] + lens[i]].tobytes() for i in range(n)]

    def counters(self):
        out = (C.c_int64 * 8)()
        _check(lib.b2_counters_read(self._h, out))
        return list(out)

    def counters_device_ptr(self):
        return lib.b2_counters_device_ptr(self._h)
