/*
 * b2rpc.h — C ABI of the B200-native brpc message-processing hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Every entry point names the
 * reference interface it replaces (paths relative to the apache/brpc tree).
 * Plain pointers and sizes only; no C++ / torch types cross this boundary.
 * All compute runs in hand-written sm_90a CUDA kernels; there is no CPU
 * fallback: every call fails with B2_E_NO_DEVICE when no CUDA device exists.
 *
 * Model.  The host messenger gathers, for each readable Socket, the bytes
 * that are pending in its read buffer (reference: Socket::_read_buf filled by
 * Socket::DoRead, src/brpc/socket.cpp:2042-2122) into one *batch*: a flat
 * byte buffer plus one b2_run per socket.  One call cuts every run into
 * messages exactly like InputMessenger::ProcessNewMessage
 * (src/brpc/input_messenger.cpp:206-322) would, decodes the RpcMeta /
 * StreamFrameMeta of each message, runs the registered device handler (echo)
 * and packs the response frames (SendRpcResponse,
 * src/brpc/policy/baidu_rpc_protocol.cpp:273-460).
 * Further down: how bytes cross PCIe (b2_set_modes: kernels pull the pinned read blocks in place, replies by reference or as the
 * writev gather list), the latency path (b2_ring_*: a persistent kernel behind a pinned submit ring), the handler set of the messenger
 * (b2_set_protocols: hulu_pbrpc / sofa_pbrpc / nshead framing; rpc_dump files as a source), leaf codecs with the reference's signatures
 * (CRC32C, snappy), the client mirror (b2_pack_requests), replies the host produced (b2_pack_responses = SendRpcResponse), and the
 * h2/gRPC server path (b2_h2_process_batch = ParseH2Message, b2_h2_pack_responses = H2UnsentResponse + PackH2Message) whose
 * per-connection state lives on the device between calls, and both halves of h2 client connections (b2_h2_pack_requests =
 * H2UnsentRequest::New + AppendAndDestroySelf; b2_h2_client_process_batch = ParseH2Message on a connected socket + what
 * ProcessHttpResponse decides; or the host parses and b2_h2_conn_peer_update mirrors the peer's SETTINGS / WINDOW_UPDATE).
 */
#ifndef B2RPC_H_
#define B2RPC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- return codes (never exceptions, never errno side channels) ---------- */
#define B2_OK              0
#define B2_E_INVAL        -1   /* bad argument */
#define B2_E_NO_DEVICE    -2   /* CUDA device/driver missing: there is NO CPU path */
#define B2_E_CUDA         -3   /* a CUDA call failed; see b2_last_error() */
#define B2_E_CAPACITY     -4   /* batch exceeds a ctx capacity (bytes / msgs / resp) */
#define B2_E_NOMEM        -5

/* ---- ParseError, identical values to src/brpc/parse_result.h:25-32 ------- */
#define B2_PARSE_OK                    0
#define B2_PARSE_ERROR_TRY_OTHERS      1
#define B2_PARSE_ERROR_NOT_ENOUGH_DATA 2
#define B2_PARSE_ERROR_TOO_BIG_DATA    3
#define B2_PARSE_ERROR_NO_RESOURCE     4
#define B2_PARSE_ERROR_ABSOLUTELY_WRONG 5

/* ---- ProtocolType subset, values of src/brpc/options.proto:38-67 --------- */
#define B2_PROTOCOL_UNKNOWN       0
#define B2_PROTOCOL_BAIDU_STD     1
#define B2_PROTOCOL_STREAMING_RPC 2
#define B2_PROTOCOL_HULU_PBRPC    3   /* framing only: b2_set_protocols */
#define B2_PROTOCOL_SOFA_PBRPC    4
#define B2_PROTOCOL_NSHEAD        12

/* ---- CompressType / ChecksumType / ContentType, options.proto:69-88 ------ */
#define B2_COMPRESS_TYPE_NONE   0
#define B2_COMPRESS_TYPE_SNAPPY 1
#define B2_COMPRESS_TYPE_GZIP   2
#define B2_COMPRESS_TYPE_ZLIB   3
#define B2_CHECKSUM_TYPE_NONE   0
#define B2_CHECKSUM_TYPE_CRC32C 1
#define B2_CONTENT_TYPE_PB      0

/* ---- brpc error codes used in replies, src/brpc/errno.proto:25-49 -------- */
#define B2_ENOSERVICE 1001
#define B2_ENOMETHOD  1002
#define B2_EREQUEST   1003
#define B2_EINTERNAL  2001
#define B2_ERESPONSE  2002

/* ---- per-message disposition (b2_msg_desc.status) ------------------------ */
#define B2_MSG_ECHOED        0  /* device handler ran, OK response packed            */
#define B2_MSG_ERROR_REPLIED 1  /* error response packed on device (error_code != 0) */
#define B2_MSG_HOST          2  /* valid request of a host-handled method; no reply  */
#define B2_MSG_BAD_META      3  /* RpcMeta failed to parse: reference closes socket
                                   with EREQUEST (baidu_rpc_protocol.cpp:577-582)   */
#define B2_MSG_STREAM_FRAME  4  /* streaming_rpc frame, meta decoded, host routes it */
#define B2_MSG_BAD_STREAM_META 5 /* StreamFrameMeta failed to parse: frame dropped
                                   (streaming_rpc_protocol.cpp:97-100)              */
#define B2_MSG_UNSUPPORTED   6  /* left to the host untouched: a non-pb content type (json ...), a reply the method wants gzip / zlib
                                   COMPRESSED, or a gzip / zlib body beyond 1 MiB (compressed or inflated; one thread walks a DEFLATE stream) */
#define B2_MSG_RESPONSE      7  /* client-side socket: a response was processed (ProcessRpcResponse,
                                   baidu_rpc_protocol.cpp:911-1013).  error_code = what Controller::SetFailed
                                   would get (0 = OK); resp_off/resp_len = the EchoResponse.message bytes,
                                   located in the BATCH buffer */
#define B2_MSG_RESPONSE_UNZ  8  /* same, the response was snappy / gzip / zlib compressed: message bytes are in the resp region */
#define B2_MSG_REPLAY       10  /* a record of an rpc_dump file (B2_RUN_RPC_DUMP) re-packed as a baidu_std request frame: resp_off/resp_len;
                                   compress_type / attachment_size = the sample's; protocol = the sample's protocol_type (only baidu_std
                                   samples are re-packed, others are B2_MSG_UNSUPPORTED) */
#define B2_MSG_FRAMED        9  /* a message of another length-prefixed protocol (hulu_pbrpc, sofa_pbrpc, nshead): cut by the
                                   device, processed by the host; protocol / frame_off / meta_size / body_size are set, body_size
                                   counts the bytes behind the 12- (hulu), 24- (sofa) or 36-byte (nshead) header */

/* ---- has_bits of b2_msg_desc --------------------------------------------- */
#define B2_HAS_REQUEST          (1u << 0)
#define B2_HAS_RESPONSE         (1u << 1)
#define B2_HAS_COMPRESS_TYPE    (1u << 2)
#define B2_HAS_CORRELATION_ID   (1u << 3)
#define B2_HAS_ATTACHMENT_SIZE  (1u << 4)
#define B2_HAS_CHUNK_INFO       (1u << 5)
#define B2_HAS_AUTH_DATA        (1u << 6)
#define B2_HAS_STREAM_SETTINGS  (1u << 7)
#define B2_HAS_USER_FIELDS      (1u << 8)
#define B2_HAS_CONTENT_TYPE     (1u << 9)
#define B2_HAS_CHECKSUM_TYPE    (1u << 10)
#define B2_HAS_CHECKSUM_VALUE   (1u << 11)
#define B2_HAS_LOG_ID           (1u << 12)
#define B2_HAS_TRACE_ID         (1u << 13)
#define B2_HAS_REQUEST_ID       (1u << 14)
#define B2_HAS_TIMEOUT_MS       (1u << 15)
/* streaming_rpc frames reuse bits 0..4: */
#define B2_SHAS_STREAM_ID        (1u << 0)
#define B2_SHAS_SOURCE_STREAM_ID (1u << 1)
#define B2_SHAS_FRAME_TYPE       (1u << 2)
#define B2_SHAS_HAS_CONTINUATION (1u << 3)
#define B2_SHAS_FEEDBACK         (1u << 4)
#define B2_SVAL_HAS_CONTINUATION (1u << 8)  /* value of has_continuation */

/*
 * One socket's pending bytes inside the batch buffer.
 * Reference: Socket::_read_buf + Socket::preferred_index()
 * (src/brpc/socket.h:865-883).  `offset` must be a multiple of 16.
 */
typedef struct b2_run {
    uint64_t socket_id;        /* opaque (SocketId); echoed back, never interpreted */
    uint32_t offset;           /* byte offset of the run inside the batch buffer */
    uint32_t length;           /* pending bytes of this socket */
    int32_t  preferred_proto;  /* Socket::preferred_index(): B2_PROTOCOL_* or -1 */
    uint32_t flags;            /* B2_RUN_* */
} b2_run;                      /* 24 bytes */
#define B2_RUN_RPC_DUMP 4u     /* the run is not a socket but an rpc_dump FILE (src/brpc/rpc_dump.cpp:237-258: records "PRPC" BE32(meta+request) BE32(meta)
                                  RpcDumpMeta request): records are cut like SampleIterator::Pop (:322-361) and every baidu_std sample is turned into the
                                  request frame rpc_replay would send (PackRpcRequest's replay branch, baidu_rpc_protocol.cpp:1067-1075): status
                                  B2_MSG_REPLAY, the frame in the resp region, correlation_id = socket_id + index of the record in the run */
#define B2_RUN_CLIENT 1u       /* Socket::CreatedByConnect(): client-side protocol rules of CutInputMessage
                                  (input_messenger.cpp:122-138) and ProcessRpcResponse instead of ProcessRpcRequest */

/*
 * Result of the cut loop for one run == what InputMessenger::ProcessNewMessage
 * leaves behind on the Socket.
 */
typedef struct b2_run_status {
    uint32_t consumed;         /* bytes cut off the front of the run (pop_front) */
    uint32_t parse_error;      /* B2_PARSE_ERROR_* that ended the loop; anything
                                  other than NOT_ENOUGH_DATA closes the socket
                                  (input_messenger.cpp:227-239) */
    uint32_t n_msgs;           /* messages cut (Socket::AddInputMessages) */
    uint32_t first_msg;        /* index of this run's first b2_msg_desc */
    int32_t  preferred_proto;  /* Socket::preferred_index() after the loop */
    uint32_t n_unanswered;     /* B2_RESP_IOVEC only (else 0): messages of this run that are NOT a device-written reply
                                  (B2_MSG_HOST, stream frames, framed-only protocols, unsupported codecs, bad metas ...), i.e.
                                  the ones the host must pick out of msgs[].  (The _avg_msg_size read-size hint,
                                  input_messenger.cpp:242-261, stays on the host: it is consumed / n_msgs smoothed.) */
    uint32_t resp_off;         /* first response byte of this run in the resp region */
    uint32_t resp_bytes;       /* span (incl. alignment padding) of this run's responses */
} b2_run_status;               /* 32 bytes */

/*
 * One cut message == MostCommonMessage (policy/most_common_message.h:33-49)
 * + the decoded RpcMeta (policy/baidu_rpc_meta.proto:26-55)
 * + where its response frame was packed.  Exactly 64 bytes, written once by
 * the device.  For B2_PROTOCOL_STREAMING_RPC frames: correlation_id =
 * StreamFrameMeta.stream_id, log_id = source_stream_id, compress_type =
 * frame_type, attachment_size = low 32 bits of feedback.consumed_size,
 * checksum_type = high 32 bits of it.
 */
typedef struct b2_msg_desc {
    uint32_t run_idx;          /* index of the b2_run this message was cut from */
    uint32_t frame_off;        /* offset of the 12-byte header in the batch buffer */
    uint32_t body_size;        /* header: meta + payload (+attachment) bytes */
    uint32_t meta_size;        /* header: RpcMeta bytes */
    int64_t  correlation_id;
    int64_t  log_id;
    int32_t  attachment_size;
    int32_t  compress_type;
    int32_t  checksum_type;
    int32_t  error_code;       /* brpc error code carried by the reply (0 = OK) */
    uint16_t has_bits;         /* B2_HAS_* */
    uint8_t  protocol;         /* B2_PROTOCOL_* */
    uint8_t  content_type;
    int16_t  method_idx;       /* registered method index, -1 = not found */
    uint16_t status;           /* B2_MSG_* */
    uint32_t resp_off;         /* offset of the reply frame in the resp region */
    uint32_t resp_len;         /* bytes of the reply frame (0 = none) */
} b2_msg_desc;                 /* 64 bytes */

/* device handler kinds for b2_register_method */
#define B2_HANDLER_HOST 0      /* descriptor only: user code runs on the host */
#define B2_HANDLER_ECHO 1      /* example::EchoService::Echo, example/echo_c++/server.cpp:44-84 */

typedef struct b2_method {
    const char* service_full_name;  /* "example.EchoService" */
    const char* service_name;       /* "EchoService" (jprotobuf short name,
                                       baidu_rpc_protocol.cpp:738-748) */
    const char* method_name;        /* "Echo" */
    const char* request_type_name;  /* "example.EchoRequest" (used in EREQUEST text) */
    int32_t handler;                /* B2_HANDLER_* */
    int32_t echo_attachment;        /* -echo_attachment (server.cpp:31) */
    int32_t response_checksum_type; /* -enable_checksum -> CRC32C (server.cpp:80-82) */
    int32_t response_compress_type; /* cntl->set_response_compress_type() */
} b2_method;

typedef struct b2_options {
    int32_t  device;           /* CUDA ordinal */
    uint32_t max_batch_bytes;  /* capacity of the device batch buffer */
    uint32_t max_msgs;         /* capacity of the descriptor array */
    uint32_t max_runs;
    uint32_t max_resp_bytes;   /* capacity of the response region (0 = derive) */
    uint32_t tile_bytes;       /* speculative scan tile, power of two (0 = default) */
    uint64_t max_body_size;    /* FLAGS_max_body_size (protocol.cpp:52), 0 = 64 MiB */
} b2_options;

/* B2_RESP_BY_REF: where reply i's payload lives.  Reply i = resp[msgs[i].resp_off, +prefix_len) followed by
 * bytes[src_off, +src_len) of the REQUEST batch — exactly how SendRpcResponse builds res_buf: header + meta, then
 * res_buf.append(res_body.movable()) / append(attachment) by reference (baidu_rpc_protocol.cpp:383-389).
 * msgs[i].resp_len = prefix_len + src_len.  src_len == 0: the whole reply is in resp (error replies, checksummed or
 * compressed replies, client-side results). */
typedef struct b2_resp_ref { uint32_t prefix_len, src_off, src_len, reserved; } b2_resp_ref;   /* 16 bytes */

/* B2_RESP_IOVEC: the same replies as ready-made `struct iovec` pairs (layout of <sys/uio.h>) with HOST addresses — what
 * IOBuf::cut_multiple_into_file_descriptor (src/butil/iobuf.cpp:954-992) assembles from the block references of the queued
 * replies before its writev, written by the GPU instead: iov[2*i] = reply i's bytes in the pinned resp block (the prefix, or the
 * whole reply), iov[2*i + 1] = its payload inside the caller's request bytes (length 0 when there is none).  A message the device
 * did not answer has two zero-length entries, so a run's replies are writev(fd, iov + 2*first_msg, 2*n_msgs) as they stand, and
 * b2_run_status.n_unanswered says whether the host has to look at that run's descriptors at all. */
typedef struct b2_iovec { void* iov_base; size_t iov_len; } b2_iovec;

/* Pointers into ctx-owned PINNED host memory, valid until the next batch call. */
typedef struct b2_batch_result {
    const b2_run_status* runs;     uint32_t n_runs;
    const b2_msg_desc*   msgs;     uint32_t n_msgs;
    const uint8_t*       resp;     uint32_t resp_bytes;   /* span of the resp region used */
    float kernel_ms;               /* device time of the kernels (CUDA events) */
    uint32_t n_launches;           /* kernels launched for this batch */
    const b2_resp_ref*   refs;     /* [n_msgs] in B2_RESP_BY_REF mode, else NULL */
    const b2_iovec*      iov;      /* [2 * n_msgs] in B2_RESP_IOVEC mode (refs is NULL then), else NULL */
} b2_batch_result;

typedef struct b2_ctx b2_ctx;

/* ---- lifecycle ----------------------------------------------------------- */
int  b2_ctx_create(const b2_options* opt, b2_ctx** out);
void b2_ctx_destroy(b2_ctx* ctx);
const char* b2_last_error(void);        /* thread-local text of the last failure */
const char* b2_version(void);

/* Replaces Server::AddService's method map used by ProcessRpcRequest
 * (FindMethodPropertyByFullName, baidu_rpc_protocol.cpp:749-756).
 * Returns the method index (>= 0) or a negative B2_E_*. */
int  b2_register_method(b2_ctx* ctx, const b2_method* m);

/* Which Protocol::parse handlers the messenger holds (InputMessenger::AddHandler, one bit per ProtocolType, probed in index order
 * exactly like CutInputMessage): default (1 << B2_PROTOCOL_BAIDU_STD) | (1 << B2_PROTOCOL_STREAMING_RPC).  The other length-prefixed
 * protocols that share MostCommonMessage can be added — ParseHuluMessage (policy/hulu_pbrpc_protocol.cpp:178-223), ParseSofaMessage
 * (policy/sofa_pbrpc_protocol.cpp:165-205), ParseNsheadMessage (policy/nshead_protocol.cpp:154-182): their messages are cut in the
 * same loop (preferred-index switching included) and surface as B2_MSG_FRAMED descriptors.  b2_run.preferred_proto may name any
 * enabled handler. */
int  b2_set_protocols(b2_ctx* ctx, uint32_t protocol_mask);

/* What the device does with streaming_rpc DATA frames beyond cutting them and decoding StreamFrameMeta:
 * B2_STREAM_DESC_ONLY (default) or B2_STREAM_SNAPPY_UNCOMPRESS — the frame payload is a snappy stream
 * (policy::SnappyDecompress(IOBuf, IOBuf), src/brpc/policy/snappy_compress.cpp:77-82, as an application of
 * example/streaming_echo_c++ would call on each received message) and is decompressed into the resp
 * region: resp_off/resp_len = the plain bytes, error_code = B2_EREQUEST when the stream is malformed. */
#define B2_STREAM_DESC_ONLY         0
#define B2_STREAM_SNAPPY_UNCOMPRESS 1
int  b2_set_stream_handler(b2_ctx* ctx, int kind);

/* "ip:port" that Controller::AppendServerIdentiy (src/brpc/controller.cpp:407-428)
 * prepends to every error text as "[ip:port]"; NULL/"" = no server identity. */
int  b2_set_server_identity(b2_ctx* ctx, const char* ip_port);

/* ---- block pool: assignable to butil::iobuf::blockmem_allocate/deallocate
 * (src/butil/iobuf.cpp:168-169), same role as rdma::block_pool
 * (src/brpc/rdma/rdma_helper.cpp:579-582, rdma/block_pool.h:74-105).  Pinned AND mapped memory, pooled: blocks
 * <= 8 KiB come from 4 MiB slabs, larger ones are cached per power-of-two class; cudaHostAlloc runs per slab, never
 * per block.  Thread-safe. ------ */
void* b2_block_alloc(size_t size);
void  b2_block_free(void* p);
uint64_t b2_block_pool_host_allocs(void);   /* cudaHostAlloc calls so far (pool diagnostics) */

/* ---- how bytes cross PCIe (both default to COPY) ---------------------------------------------------------
 * input:  B2_INPUT_COPY  cudaMemcpyAsync of the batch bytes into HBM, kernels read HBM.
 *         B2_INPUT_PULL  `bytes` of every batch call MUST be memory from b2_block_alloc (pinned + mapped; the socket
 *                        read blocks themselves, like the RDMA transport's registered blocks): the kernels read it IN
 *                        PLACE over PCIe, so only what the parse touches crosses the link — frame headers, RpcMeta, the
 *                        first body bytes, the speculative scan windows; bodies only when a checksum / codec needs them.
 * resp:   B2_RESP_COPY   every reply frame is materialised in the resp region and copied back.
 *         B2_RESP_BY_REF an OK echo reply is {prefix in resp, payload = a span of the request bytes} (b2_resp_ref), what
 *                        SendRpcResponse does with IOBuf references; only descriptors, refs and <= 64-byte prefixes
 *                        come back.  Everything else (errors, CRC'd / compressed replies) is still materialised.
 *         B2_RESP_IOVEC  BY_REF with the references already turned into the iovec list of the write (b2_iovec): the host
 *                        side does no per-message work for device-answered traffic. */
#define B2_INPUT_COPY 0
#define B2_INPUT_PULL 1
#define B2_RESP_COPY   0
#define B2_RESP_BY_REF 1
#define B2_RESP_IOVEC  2   /* BY_REF, and the device also writes the gather list: b2_batch_result.iov (below) */
int  b2_set_modes(b2_ctx* ctx, int input_mode, int resp_mode);

/* ---- the hot path, host-facing (H2D + kernels + D2H inside) ---------------
 * Replaces, for every run: InputMessenger::ProcessNewMessage
 * (input_messenger.cpp:206-322) -> CutInputMessage (:84-179) ->
 * ParseRpcMessage / ParseStreamingMessage -> ProcessRpcRequest
 * (baidu_rpc_protocol.cpp:568-866) -> SendRpcResponse (:273-460).
 * `bytes` may be any host memory (pinned memory from b2_block_alloc avoids a
 * staging copy). */
int  b2_process_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes,
                      const b2_run* runs, uint32_t n_runs, b2_batch_result* out);

/* b2_process_batch split in two so that several batches (one ctx each) can be in flight on
 * one GPU: submit enqueues H2D + kernels on the ctx's stream and returns; collect waits and
 * brings descriptors + responses back.  With >= 3 contexts the H2D copy of one batch, the
 * kernels of another and the D2H copy of a third overlap (full-duplex PCIe). */
int  b2_batch_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs);
int  b2_batch_collect(b2_ctx* ctx, b2_batch_result* out);

/* ---- the latency path: a PERSISTENT kernel per context fed through a submit ring (north star: "a persistent per-GPU kernel
 * pulls batches of raw socket bytes staged into pinned host IOBuf blocks") -----------------------------------------------
 * For batches of up to 128 KiB / 512 runs / 1024 messages — what a set of synchronous clients keeps in flight — there is no
 * kernel launch, no cudaMemcpy and no stream synchronisation per batch: b2_ring_submit fills a slot of a ring that lives in
 * pinned + mapped host memory and rings its doorbell with a plain store; the resident kernel (one CTA, started by
 * b2_ring_start or by the first submission) polls the doorbell over PCIe, pulls runs and bytes (in place when `bytes` is
 * b2_block_alloc memory, else from the slot's staging copy), runs the same cut / decode / echo / pack code as
 * b2_process_batch and writes descriptors + replies straight into the slot's pinned output block; b2_ring_wait spins on the
 * slot's completion word.  Same role as the RDMA transport's always-polling completion loop (RdmaEndpoint::PollCq,
 * src/brpc/rdma/rdma_endpoint.cpp:1470-1591).  Up to 8 tickets may be in flight; a result stays valid until 8 further
 * submissions.  The kernel retires after 20 ms without work (B2_RING_IDLE_MS) so that it never blocks device-wide
 * synchronisation for long, and comes back with the next submission.  A batch whose results do not fit the compact block is
 * served by the big pipeline inside b2_ring_wait (needs every other ticket collected).  Not to be mixed with concurrent
 * batch calls on the same context.
 * With a stream table and b2_stream_ring_enable the ring also runs the stream pass (below) after each ticket's batch, in the same
 * kernel, and each slot carries the ticket's stream results.  On such a context tickets are collected in ticket order
 * (b2_ring_wait of any other ticket fails with B2_E_INVAL), and a ticket that overflows the compact block keeps its place: the
 * kernel runs no pass for it and parks before the next ticket until b2_ring_wait has served it through the big pipeline (stream
 * pass included) and released the kernel through a control word; the tickets behind it need not be collected first. */
int  b2_ring_start(b2_ctx* ctx);
int  b2_ring_stop(b2_ctx* ctx);
int  b2_ring_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs, uint32_t* ticket);
int  b2_ring_wait(b2_ctx* ctx, uint32_t ticket, b2_batch_result* out);
uint64_t b2_ring_launches(b2_ctx* ctx);   /* how many times the resident kernel was (re)started: the launches of the ring path */
/* Device-side phases of a collected ticket (diagnostics), nanoseconds since the resident kernel saw the doorbell:
 * [0] slot header read, [1] runs + bytes pulled into HBM, [2] cut / decode / echo / pack done, [3] results pushed to the host. */
int  b2_ring_phase_ns(b2_ctx* ctx, uint32_t ticket, uint64_t out[4]);
/* Measurement helper: us_out[i] = wall-clock microseconds of the i-th of `iters` back-to-back single-batch calls —
 * b2_process_batch (use_ring 0) or b2_ring_submit + b2_ring_wait (use_ring 1) — timed inside the library. */
int  b2_latency_probe(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                      uint32_t iters, int use_ring, float* us_out);

/* ---- the same path split in three, for measurement with inputs resident in
 * HBM (bench.py `value`): upload once, execute many times, download. -------- */
int  b2_batch_upload(b2_ctx* ctx, const void* bytes, uint32_t nbytes,
                     const b2_run* runs, uint32_t n_runs);
int  b2_batch_execute(b2_ctx* ctx, float* kernel_ms, uint32_t* n_launches);
int  b2_batch_download(b2_ctx* ctx, b2_batch_result* out);
/* `steps` back-to-back passes of the whole kernel pipeline over the resident batch,
 * one CUDA-event pair around all of them on the launching stream. */
int  b2_batch_execute_many(b2_ctx* ctx, uint32_t steps, float* total_ms, uint32_t* n_launches);

/* Asynchronous form for pipelining several resident batches (one ctx each) on one GPU:
 * b2_batch_launch enqueues one pass on the ctx's stream and returns; b2_batch_wait blocks
 * until it is done.  b2_elapsed_ms(a, b) = device time from a's FIRST launch since its last
 * wait to b's LAST launch end (CUDA events; a and b may be the same ctx).  A launched pass records no stage events: b2_stage_times reports
 * none after it, and kernel_ms keeps the value of the last executed or collected batch. */
int  b2_batch_launch(b2_ctx* ctx);
int  b2_batch_wait(b2_ctx* ctx);
int  b2_elapsed_ms(b2_ctx* a, b2_ctx* b, float* ms);

/* What the last upload / launch decided: out[0] tile bytes, [1] tiles, [2] frame offsets kept per tile, [3] 1 = the fused
 * decode+pack kernel served the batch (0 = the slot-scan pipeline). */
int  b2_batch_info(b2_ctx* ctx, uint32_t out[4]);

/* Walk groups of the front stages (DESIGN §3): k_tile_search finds a speculative entry only in the first tile of each group of
 * consecutive tiles of a connection, and one thread of k_tile_walk walks the frame chain across the whole group.  mode 0 (default) =
 * auto: 2 tiles per group on the fused path once the frame size is known and frames are not small enough to take the dense shape, 1
 * elsewhere; 1 = one tile per group (every tile searched); 2..8 = that many tiles per group on every path but B2_INPUT_PULL.  Results
 * do not depend on it.  Takes effect at the next upload (an uploaded batch has to be uploaded again).  b2_walk_group returns the
 * group size the last launch used. */
int  b2_set_walk_group(b2_ctx* ctx, uint32_t mode);
int  b2_walk_group(b2_ctx* ctx);

/* Residency of a fused pass.  Two contexts on two streams overlap their passes: one batch's front stages (k_tile_search, k_tile_walk,
 * k_resolve) and slow-reply kernel (k_pack_slow<true>) run on the SMs the other batch's k_fused holds, which they can only do where one
 * of their blocks fits in what a k_fused CTA leaves of the SM.  Entry 0 is k_fused in the shape the uploaded batch uses, then those four
 * kernels as launched: registers per thread and static shared memory from the compiled kernels, threads per block, shared memory per
 * block including the dynamic part for the uploaded batch, and `fits`, the number of blocks an SM holding one k_fused CTA can start
 * beside it (registers allocated 256 per warp; the shared memory the SM is configured with for the k_fused CTA, in the device's steps,
 * less the CTA's own and each block's reserve; warp and block slots).  Writes up to `cap` entries and returns the number of kernels (5). */
typedef struct b2_resident_kernel {
    const char* name;
    uint32_t regs, threads, smem_bytes, fits;
} b2_resident_kernel;   /* 24 bytes */
int  b2_resident_plan(b2_ctx* ctx, b2_resident_kernel* out, int cap);

/* PCI bus id ("0000:1b:00.0") of a device, for a host side that wants to run its polling threads and first-touch its pinned blocks on
 * the CPUs next to the GPU (/sys/bus/pci/devices/<id>/local_cpulist): zero-copy reads that cross the socket interconnect lose most of
 * their rate.  No ctx needed.  (brpc pins nothing itself; its RDMA endpoint leaves NUMA placement to the deployment as well.) */
int  b2_device_pci_bus_id(int device, char* out, int cap);

/* Device time of each stage of the last execute, in launch order.  Writes up to
 * `cap` entries of (name, ms); returns the number of stages. */
int  b2_stage_times(b2_ctx* ctx, const char** names, float* ms, int cap);

/* ---- leaf codecs on device-resident or host buffers ----------------------
 * b2_crc32c_batch: one CRC-32C per (offset,length) slice == butil::crc32c::Value
 * (src/butil/crc32c.h:30-33) on each slice; out[i] is the UNMASKED crc. */
int  b2_crc32c_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes,
                     const uint32_t* offs, const uint32_t* lens, uint32_t n,
                     uint32_t* out);

/* b2_snappy_uncompress_batch: butil::snappy::Uncompress (src/butil/third_party/snappy/snappy.cc:1526-1552)
 * on each (offset,length) slice of raw-format snappy.  Output i is written to out + out_offs[i]
 * (out_offs is filled by the call, 16-byte aligned, in slice order) and out_lens[i] is its length,
 * or -1 when the reference would return false (malformed stream / length mismatch). */
int  b2_snappy_uncompress_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes,
                                const uint32_t* offs, const uint32_t* lens, uint32_t n,
                                void* out, uint32_t out_cap, uint32_t* out_offs, int32_t* out_lens);

/* b2_snappy_compress_batch: butil::snappy::Compress (snappy.cc:875-956), BIT-EXACT with the vendored
 * 1.1.3 encoder, on each (offset,length) slice.  Output i goes to out + out_offs[i] (filled by the
 * call: slots of MaxCompressedLength, 16-byte aligned), out_lens[i] = compressed size. */
int  b2_snappy_compress_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes,
                              const uint32_t* offs, const uint32_t* lens, uint32_t n,
                              void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens);

/* ---- the same leaves with the REFERENCE's own signatures, for direct substitution at seam 4 (the bodies of the
 * CompressHandler / ChecksumHandler registered in src/brpc/global.cpp:400-418, or any direct caller):
 *   b2_crc32c_extend                  == butil::crc32c::Extend          (src/butil/crc32c.h:24)
 *   b2_snappy_max_compressed_length   == butil::snappy::MaxCompressedLength   (third_party/snappy/snappy.h:112)
 *   b2_snappy_raw_compress            == butil::snappy::RawCompress     (snappy.h:125)   bit-exact output
 *   b2_snappy_get_uncompressed_length == butil::snappy::GetUncompressedLength (snappy.h:141), returns 1/0 for true/false
 *   b2_snappy_raw_uncompress          == butil::snappy::RawUncompress   (snappy.h:135), returns 1/0
 * They run on a process-wide default context (device $B2_DEVICE, default 0), one buffer per call: correct, not fast — the
 * batch forms above are the throughput path. */
uint32_t b2_crc32c_extend(uint32_t init_crc, const char* data, size_t n);
size_t   b2_snappy_max_compressed_length(size_t source_bytes);
void     b2_snappy_raw_compress(const char* input, size_t input_length, char* compressed, size_t* compressed_length);
int      b2_snappy_get_uncompressed_length(const char* compressed, size_t compressed_length, size_t* result);
int      b2_snappy_raw_uncompress(const char* compressed, size_t compressed_length, char* uncompressed);

/* ---- client mirror (SURVEY §8a a13 / a14): PackRpcRequest (src/brpc/policy/baidu_rpc_protocol.cpp:1045-1133) with
 * SerializeRpcRequest (:1015-1043: EchoRequest{message}, COMPRESS_TYPE_NONE / SNAPPY, CRC32C over the serialized body)
 * and PackStreamMessage (policy/streaming_rpc_protocol.cpp:42-58), one warp per frame.  RpcRequestMeta carries the
 * registered method's service_full_name / method_name (-baidu_protocol_use_fullname=true), log_id and timeout_ms when
 * flagged; RpcMeta always carries compress_type, correlation_id, content_type(0), checksum_type and checksum_value (what
 * PackRpcRequest sets unconditionally) and attachment_size when there is an attachment.  Tracing fields and request_id
 * are not covered.  Frame i lands at out + out_offs[i] (filled by the call), out_lens[i] long (0 = could not be packed). */
#define B2_REQ_BAIDU_STD     0
#define B2_REQ_STREAM_FRAME  1
#define B2_REQ_HAS_LOG_ID            1u   /* baidu_std */
#define B2_REQ_HAS_TIMEOUT           2u   /* baidu_std: timeout_ms > 0 is written */
#define B2_REQ_HAS_SOURCE_STREAM_ID  1u   /* stream frame */
#define B2_REQ_HAS_CONTINUATION      2u   /* stream frame: has_continuation is present ... */
#define B2_REQ_CONTINUATION_VALUE    4u   /* ... with this value */
typedef struct b2_request {
    uint32_t kind, flags;
    int32_t  method_idx;             /* baidu_std: registered method */
    int32_t  timeout_ms;             /* baidu_std */
    int64_t  correlation_id;         /* stream frame: stream_id */
    int64_t  log_id;                 /* stream frame: source_stream_id */
    int32_t  compress_type, checksum_type;   /* baidu_std */
    int32_t  frame_type;             /* stream frame: brpc::FrameType */
    uint32_t payload_off, payload_len;        /* EchoRequest.message / the stream data */
    uint32_t attachment_off, attachment_len;  /* baidu_std */
    uint32_t reserved;
} b2_request;                        /* 64 bytes */
int  b2_pack_requests(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_request* reqs, uint32_t n,
                      void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens);
/* baidu_std CLIENT connections on the latency path: b2_process_batch followed by b2_pack_requests inside the resident k_ring
 * (k_ring<RingBody::requests>) fed through the same submit ring.  A ticket is one turn of a client's event loop: read what arrived, then send what is
 * queued.  The runs (the bytes read from client sockets, B2_RUN_CLIENT) are served as by b2_ring_submit, then the requests are packed as
 * by b2_pack_requests; their fields index the same `bytes` as the runs.  A baidu_std client keeps no connection state on the device
 * (correlation ids live on the host), so a ticket's requests do not depend on its runs: they are packed even when the runs overflow the
 * compact block.  Runs are served whatever their flags: server runs in a client ticket are answered as b2_ring_submit answers them.
 * For each socket hand its reads over first, then write its request frames in request order.
 * A context runs one ring kind: b2_ring_submit / _wait, b2_stream_ring_enable, b2_ring_turn_* and the b2_h2_*ring* calls refuse a
 * context that runs this one, and b2_client_ring_* refuse a context of another kind.
 * b2_client_ring_enable: once, before the context's first ring call, and not on a context with a stream table (else B2_E_INVAL; the
 * ticket runs no stream pass).  max_bytes bounds a ticket's whole `bytes` (the runs' bytes plus the request payloads, <= max_batch_bytes,
 * so a turn may exceed b2_ring_submit's 128 KiB); max_reqs (<= max_msgs) and req_out_cap (<= max_resp_bytes) play the roles of
 * b2_pack_requests' n and out_cap.  Caps above those limits fail with B2_E_CAPACITY; they fix the slot layout.
 * b2_ring_stop, b2_ring_launches, b2_ring_phase_ns ([2]: runs served and requests packed) and B2_RING_IDLE_MS apply as to k_ring.
 * b2_client_ring_submit: n_runs or n_reqs may be 0, not both.  Every check of b2_ring_submit (<= 512 runs, 16-aligned runs inside
 * `bytes`) and of b2_pack_requests (payloads inside `bytes`, every frame placed at its worst-case size within req_out_cap) applies with
 * the enable-time caps; a failed check claims no slot and leaves the next ticket number unchanged.  The runs keep the compact block's
 * limits (1024 messages, its reply bytes), sized from the extent the runs cover.  Bytes in b2_block_alloc memory are pulled in place,
 * others staged into the slot.
 * b2_client_ring_wait: tickets may be waited in any order.  For every ticket `batch` equals b2_process_batch(bytes, runs) on a context
 * with the same settings, and the request offsets, lengths and frame bytes equal b2_pack_requests(bytes, reqs, req_out_cap) — for any
 * sequence of tickets, byte for byte.  A ticket whose runs overflow the compact block has them served through the big pipeline inside the
 * wait, as b2_ring_wait does (every other ticket collected first); its frames still come from the kernel.  B2_RESP_BY_REF / B2_RESP_IOVEC
 * behave as in b2_ring_wait.  While a ticket is outstanding every call that uploads to the context (b2_process_batch, b2_batch_*,
 * b2_pack_requests, b2_pack_responses, the crc32c / snappy / hpack / h2 calls, b2_stream_write) fails with B2_E_INVAL. */
typedef struct b2_client_ring_result {   /* views into the ticket's pinned slot, valid until the 8th later submission */
    b2_batch_result batch;               /* the runs, exactly as b2_ring_wait returns them */
    uint32_t n_reqs, reserved;
    const uint32_t* req_offs;            /* as b2_pack_requests' out_offs */
    const uint32_t* req_lens;            /* as its out_lens: 0 = could not be packed */
    const uint8_t*  req_out;             /* request i's frame at req_out + req_offs[i] */
} b2_client_ring_result;                 /* 104 bytes */
int  b2_client_ring_enable(b2_ctx* ctx, uint32_t max_bytes, uint32_t max_reqs, uint32_t req_out_cap);
int  b2_client_ring_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                           const b2_request* reqs, uint32_t n_reqs, uint32_t* ticket);
int  b2_client_ring_wait(b2_ctx* ctx, uint32_t ticket, b2_client_ring_result* out);

/* ---- replies the HOST produced (B2_HANDLER_HOST methods, any service above the transport): SendRpcResponse
 * (src/brpc/policy/baidu_rpc_protocol.cpp:273-460) as a batch, one warp per reply.  `bytes` holds what the host has: the response
 * message as its Serializer wrote it (UNcompressed), the attachment, the error text, the request's checksum bytes, user fields.
 *   - body: SerializeResponse (:218-246) -> SerializeRpcMessage (:148-216): COMPRESS_TYPE_NONE copies it, SNAPPY compresses it here
 *     (bit-exact with the vendored snappy); response_checksum_type CRC32C is computed here over the (compressed) body
 *     (Crc32cCompute, policy/crc32c_checksum.cpp:28-42).  gzip / zlib replies are not packed (out_lens[i] = 0): bit-exact deflate
 *     output is zlib-version specific.
 *   - error_code != 0 (cntl->Failed()): no body, no attachment, nothing compressed or checksummed (:316-330); -1 becomes
 *     EINTERNAL (:333-337); error_text is written only when non-empty (:343-347).
 *   - RpcMeta (:339-380): response{error_code,[error_text]}, compress_type, correlation_id, [attachment_size], [stream_settings
 *     {stream_id, need_feedback, writable, extra_stream_ids}] (Stream::FillSettings, stream.cpp:678-682), [user_fields], content_type,
 *     checksum_type, checksum_value.  checksum_value = the CRC when one was computed, else the bytes at checksum_value_off — the
 *     REQUEST's checksum_value, which the Controller still holds (:608 + :349).  user_fields are written in the order given (a
 *     protobuf map has no defined wire order; with one entry there is nothing to order).
 * Reply i lands at out + out_offs[i] (filled by the call), out_lens[i] long (0 = could not be packed). */
#define B2_RSP_HAS_STREAM         1u
#define B2_RSP_STREAM_NEED_FEEDBACK 2u
#define B2_RSP_STREAM_WRITABLE    4u
typedef struct b2_reply {
    uint32_t flags;
    int32_t  error_code;
    int64_t  correlation_id;
    int32_t  compress_type, checksum_type, content_type;
    uint32_t error_text_off, error_text_len;
    uint32_t body_off, body_len;
    uint32_t attachment_off, attachment_len;
    uint32_t checksum_value_off, checksum_value_len;
    uint32_t extra_streams_off, n_extra_streams;   /* int64 little-endian each, 8-byte aligned offset */
    uint32_t user_fields_off, n_user_fields;       /* records: u32 key_len, u32 value_len, key bytes, value bytes (unaligned, back to back) */
    uint32_t reserved;
    int64_t  stream_id;
} b2_reply;                          /* 88 bytes */
int  b2_pack_responses(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_reply* replies, uint32_t n,
                       void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens);
/* baidu_std SERVER turns on the latency path: b2_process_batch followed by b2_pack_responses inside the resident k_ring
 * (k_ring<RingBody::replies>) fed through the same submit ring.  A ticket is one turn of a server's event loop: read what arrived, then
 * send the replies user code produced for B2_HANDLER_HOST methods since the last turn.  The runs are served as by b2_ring_submit (device
 * methods are answered in the compact block as before), then the replies are packed as by b2_pack_responses; their fields index the same
 * `bytes` as the runs.  A baidu_std server keeps no connection state on the device, so a turn's replies do not depend on its runs: they
 * are packed even when the runs overflow the compact block.  baidu_std clients match replies by correlation_id, so the order in which
 * the host writes a socket's device-answered replies and its host replies does not matter.
 * A context runs one ring kind: b2_ring_submit / _wait, b2_stream_ring_enable, b2_client_ring_* and the b2_h2_*ring* calls refuse a
 * context that runs this one, and b2_ring_turn_* refuse a context of another kind.
 * b2_ring_turn_enable: once, before the context's first ring call, and not on a context with a stream table (else B2_E_INVAL; the turn
 * runs no stream pass: a reply that accepts a Stream goes through the batch calls).  Every cap must be non-zero (else B2_E_INVAL).
 * max_bytes bounds a turn's whole `bytes` (the runs' bytes plus the reply bodies, <= max_batch_bytes, so a turn may exceed
 * b2_ring_submit's 128 KiB); max_resps (max_resps * 88 <= max_msgs * 64, as for b2_pack_responses' n) and resp_out_cap
 * (<= max_resp_bytes) play the roles of b2_pack_responses' n and out_cap.  Caps above those limits fail with B2_E_CAPACITY; they fix the
 * slot layout.  b2_ring_stop, b2_ring_launches, b2_ring_phase_ns ([2]: runs served and replies packed) and B2_RING_IDLE_MS apply as
 * to k_ring.
 * b2_ring_turn_submit: n_runs or n_replies may be 0, not both.  Every check of b2_ring_submit (<= 512 runs, 16-aligned runs inside
 * `bytes`) and of b2_pack_responses (reply fields inside `bytes`, every frame placed at its worst-case size within resp_out_cap) applies
 * with the enable-time caps and the same codes; a failed check claims no slot and leaves the next ticket number unchanged.  The runs keep
 * the compact block's limits (1024 messages, its reply bytes), sized from the extent the runs cover.  Bytes in b2_block_alloc memory are
 * pulled in place, others staged into the slot.
 * b2_ring_turn_wait: tickets may be waited in any order.  For any sequence of turns `batch` equals b2_process_batch(bytes, runs), and
 * each reply's offset, length and frame bytes equal b2_pack_responses(bytes, replies, resp_out_cap), on a context with the same settings,
 * byte for byte.  gzip / zlib replies come back with length 0, as from b2_pack_responses.  A turn whose runs overflow the compact block has
 * them served through the big pipeline inside the wait, as b2_ring_wait does (every other ticket collected first); its replies still come
 * from the kernel.  B2_RESP_BY_REF / B2_RESP_IOVEC apply to the runs only, as in b2_ring_wait.  While a turn is outstanding every call
 * that uploads to the context (b2_process_batch, b2_batch_*, b2_pack_requests, b2_pack_responses, the crc32c / snappy / hpack / h2
 * calls) fails with B2_E_INVAL. */
typedef struct b2_ring_turn_result {     /* views into the ticket's pinned slot, valid until the 8th later submission */
    b2_batch_result batch;               /* the runs, exactly as b2_ring_wait returns them */
    uint32_t n_replies, reserved;
    const uint32_t* reply_offs;          /* as b2_pack_responses' out_offs */
    const uint32_t* reply_lens;          /* as its out_lens: 0 = could not be packed */
    const uint8_t*  reply_out;           /* reply i's frame at reply_out + reply_offs[i] */
} b2_ring_turn_result;                   /* 104 bytes */
int  b2_ring_turn_enable(b2_ctx* ctx, uint32_t max_bytes, uint32_t max_resps, uint32_t resp_out_cap);
int  b2_ring_turn_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                         const b2_reply* replies, uint32_t n_replies, uint32_t* ticket);
int  b2_ring_turn_wait(b2_ctx* ctx, uint32_t ticket, b2_ring_turn_result* out);

/* ---- h2 / gRPC (SURVEY §8a a15): leaf calls first, then the whole server-side parser and the reply framing -----
 * b2_h2_scan_batch: H2Context::ConsumeFrameHead (src/brpc/policy/http2_rpc_protocol.cpp:438-465)
 * chained over every connection run.  runs[i].flags & B2_RUN_H2_PREFACE: the run starts a server-side
 * connection, the 24-byte client preface (:119-120, :469-479) is checked and skipped first.
 * frames of run i land at frames[i * cap_per_run ...]; err[i] is a B2_PARSE_ERROR_*. */
#define B2_RUN_H2_PREFACE 2u
typedef struct b2_h2_frame { uint8_t type, flags; uint16_t pad; uint32_t stream_id, payload_off, payload_len; } b2_h2_frame;
int  b2_h2_scan_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                      uint32_t max_frame_size, b2_h2_frame* frames, uint32_t cap_per_run,
                      uint32_t* n_frames, uint32_t* consumed, uint32_t* err);
/* b2_hpack_decode_batch: HPacker::Decode (src/brpc/details/hpack.cpp:765-843) looped over header
 * blocks like H2StreamContext::ConsumeHeaders (http2_rpc_protocol.cpp:1221-1232).  Blocks of one
 * connection must be adjacent and in wire order; every connection (0 .. B2_HPACK_MAX_CONNS-1) owns a
 * dynamic table that persists across calls (b2_hpack_reset starts a new connection).  Block i's
 * records (u16 name_len, u16 value_len, name, value) land at out + i * per_block_cap.
 * status[i]: 0 consumed, 1 ran out of bytes inside a field, -1 malformed, -2 per_block_cap exceeded. */
#define B2_HPACK_MAX_CONNS 4096
typedef struct b2_hpack_block { uint32_t conn, offset, length, reserved; } b2_hpack_block;
int  b2_hpack_reset(b2_ctx* ctx, uint32_t conn, uint32_t max_table_size);
int  b2_hpack_decode_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_hpack_block* blocks, uint32_t n_blocks,
                           void* out, uint32_t per_block_cap, uint32_t* out_lens, int32_t* status, uint32_t* n_headers);

/* b2_h2_process_batch: the server side of ParseH2Message (src/brpc/policy/http2_rpc_protocol.cpp:1103-1138) =
 * H2Context::Consume (:467-543) looped over every connection run: client preface, frame heads, the frame handlers
 * OnData/OnHeaders/OnContinuation/OnResetStream/OnSettings/OnPing/OnGoAway/OnWindowUpdate (:545-1041) with their
 * flow-control bookkeeping, H2StreamContext::ConsumeHeaders (:1221-1306) over the connection's HPACK table, and — for
 * every stream that reaches OnEndStream — what ProcessHttpRequest reads first: ParseContentType and RemoveGrpcPrefix
 * (policy/http_rpc_protocol.cpp:176-230, :264-277) and the "/service/method" lookup of FindMethodPropertyByURIImpl
 * (:1088-1138, plain service/method form only).
 *   runs[i].socket_id = connection index (0 .. B2_H2_MAX_CONNS-1); state (settings, windows, pending streams, HPACK
 *   table) persists across calls; b2_h2_conn_reset starts a new server-side connection (H2Context ctor + Init).
 *   rs[i].ctrl_off/len  : the bytes the reference WriteAck()s while parsing (SETTINGS + WINDOW_UPDATE after the
 *                         preface, SETTINGS acks, PING acks, RST_STREAM, GOAWAY, WINDOW_UPDATEs), in order, inside out.
 *   msgs                : one per completed request, in parse order per run; header records (u16 name_len,
 *                         u16 value_len, name, value — every decoded field in order) and the concatenated DATA
 *                         payloads live in out.
 * Device capacities (the reference has none; they are run-time choices, b2_h2_configure): `max_pending` concurrent unfinished
 * streams per connection and `stream_bytes` (4 KiB of header records + the body) per unfinished stream whose body spans
 * several DATA frames (a body carried by one DATA frame is referenced in the input and needs none); beyond them the run ends
 * with B2_PARSE_ERROR_NO_RESOURCE (the host takes the connection over or closes it, input_messenger.cpp:227-239).
 * Defaults: B2_H2_MAX_CONNS connections x B2_H2_MAX_PENDING streams x B2_H2_STREAM_BYTES.  gRPC clients keep up to 100
 * calls in flight per connection (the server side of brpc advertises no SETTINGS_MAX_CONCURRENT_STREAMS): size
 * max_pending for that, e.g. b2_h2_configure(ctx, 256, 128, 69632) = 2.2 GB of the 80 GB HBM. */
#define B2_H2_MAX_CONNS 1024
#define B2_H2_MAX_PENDING 8
#define B2_H2_STREAM_BYTES 69632
/* Must precede the first h2 call on the context (the pool is allocated then).  stream_bytes: multiple of 16, > 4 KiB. */
int  b2_h2_configure(b2_ctx* ctx, uint32_t max_conns, uint32_t max_pending, uint32_t stream_bytes);
#define B2_H2_HEADER_BYTES 4096
#define B2_H2_FLAG_GRPC            1u   /* content-type is application/grpc[+...] (is_grpc_ct) */
#define B2_H2_FLAG_GRPC_PREFIX_OK  2u   /* RemoveGrpcPrefix succeeded: msg_off/msg_len are valid */
#define B2_H2_FLAG_GRPC_COMPRESSED 4u   /* compressed flag of the 5-byte prefix */
#define B2_H2_FLAG_HAS_PATH        8u
#define B2_H2_FLAG_BODY_IN_INPUT  16u   /* body_off/msg_off index the INPUT bytes (a single DATA frame carried the whole body): zero copy */
#define B2_H2_NO_METHOD 255u            /* no :method header (HttpHeader defaults to GET) */
typedef struct b2_h2_run_status {
    uint32_t consumed, parse_error, n_msgs, first_msg;
    uint32_t ctrl_off, ctrl_len;
    uint32_t remote_max_frame_size, remote_stream_window_size;   /* what PackH2Message needs next */
} b2_h2_run_status;                                              /* 32 bytes */
typedef struct b2_h2_msg {
    uint32_t run_idx, stream_id;
    uint32_t headers_off, headers_len, n_headers;
    uint32_t body_off, body_len;
    uint32_t http_method;        /* brpc::HttpMethod of the last :method, B2_H2_NO_METHOD if none */
    uint32_t content_type;       /* brpc::HttpContentType of the last content-type header (0 = others / none) */
    uint32_t flags;              /* B2_H2_FLAG_* */
    int32_t  method_idx;         /* registered method named by :path, -1 if none */
    uint32_t msg_off, msg_len;   /* gRPC message (body without the 5-byte prefix) */
    uint32_t path_off, path_len; /* the path part of :path inside out */
    uint32_t reserved;
} b2_h2_msg;                     /* 64 bytes */
int  b2_h2_conn_reset(b2_ctx* ctx, uint32_t conn);
int  b2_h2_process_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                         b2_h2_run_status* rs, b2_h2_msg* msgs, uint32_t msg_cap, uint32_t* n_msgs,
                         void* out, uint32_t out_cap);

/* b2_h2_pack_responses: H2UnsentResponse::AppendAndDestroySelf (src/brpc/policy/http2_rpc_protocol.cpp:1688-1750) +
 * PackH2Message (:1310-1380) + AddGrpcPrefix (policy/http_rpc_protocol.cpp:254-262) for a list of responses:
 * connection flow control (MinusWindowSize, else RST_STREAM(FLOW_CONTROL_ERROR)), HPacker::Encode (details/hpack.cpp:696-726)
 * of ":status" and "content-type" — and of the "grpc-status" / "grpc-message" trailers of a gRPC response — against
 * the connection's ENCODER table (indexed if present, else literal with incremental indexing and a name index when one
 * exists, no Huffman: the reference's defaults; never-indexed when the peer announced header_table_size 0), HEADERS
 * (+CONTINUATION), DATA frames split at the peer's max_frame_size, trailers, and the deferred connection WINDOW_UPDATE.
 * Responses of one connection must be adjacent and in write order; the state is the connection's (b2_h2_process_batch).
 * Response i's bytes land at out + out_offs[i] (filled by the call), out_lens[i] long.  User-defined response headers
 * are not covered.  bytes may be NULL (nbytes 0) when every field uses a zero-copy source. */
#define B2_H2_RESP_GRPC 1u
/* zero-copy sources: the buffers of the LAST b2_h2_process_batch on this context are still on the device.  A later call that
 * overwrites the context's device input ends that, b2_ring_submit included (k_ring pulls every ticket there): the flags are then
 * refused with B2_E_INVAL. */
#define B2_H2_RESP_BODY_IN_INPUT 2u   /* body_off indexes that call's input bytes (e.g. an echoed B2_H2_FLAG_BODY_IN_INPUT message) */
#define B2_H2_RESP_BODY_IN_OUT   4u   /* body_off indexes that call's out buffer */
#define B2_H2_RESP_CT_IN_OUT     8u   /* content_type_off indexes that call's out buffer (the request's own content-type value) */
typedef struct b2_h2_response {
    uint32_t conn, stream_id;
    int32_t  status_code;                            /* :status */
    uint32_t flags;                                  /* B2_H2_RESP_GRPC */
    uint32_t content_type_off, content_type_len;     /* inside bytes; length 0 = no content-type header */
    uint32_t body_off, body_len;                     /* the body; for gRPC the serialized message (the prefix is added here) */
    int32_t  grpc_status;
    uint32_t grpc_message_off, grpc_message_len;     /* already percent-encoded; length 0 = none */
    uint32_t reserved;
} b2_h2_response;                                    /* 48 bytes */
int  b2_h2_pack_responses(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_h2_response* resps, uint32_t n,
                          void* out, uint32_t out_cap, uint32_t* out_offs, uint32_t* out_lens);

/* b2_h2_pack_requests — the CLIENT side of the same connection state: H2UnsentRequest::New (src/brpc/policy/http2_rpc_protocol.cpp:
 * 1382-1453: the header list) + H2UnsentRequest::AppendAndDestroySelf (:1496-1592) + PackH2Message (:1310-1380), what PackH2Request
 * (:1784-1800) queues for a call on an "h2" / "h2:grpc" channel.  Per request, in the reference's order:
 *   - the first request of a connection (b2_h2_conn_reset, nothing packed yet) is preceded by the 24-byte client preface and
 *     SerializeH2SettingsFrameAndWU of the default client settings (:253-265, flags :34-43: ENABLE_PUSH 0, INITIAL_WINDOW_SIZE 256 KiB,
 *     connection WINDOW_UPDATE 1 MiB - 65535) — written even when the request itself is then refused, as `out` has them there;
 *   - AllocateClientStreamId (http2_rpc_protocol.h:399-412): 1, 3, 5, ...; past 0x7fffffff -> B2_H2_REQ_RUNOUT (EH2RUNOUTSTREAMS);
 *   - a non-empty body is charged to the flow-control windows (H2StreamContext::ConsumeWindowSize :1199-1219): the peer's initial stream
 *     window, then MinusWindowSize on the connection window; not enough -> B2_H2_REQ_ELIMIT, the stream id stays consumed;
 *   - HPacker::Encode (details/hpack.cpp:696-726) against the connection's encoder table of ":method" (POST, or GET with
 *     B2_H2_REQ_GET), ":scheme" (http / https), ":path", ":authority", "content-type" when non-empty, "accept: * / *" and
 *     "user-agent: brpc/1.0 curl/7.0" when the flags say the call set neither (need_accept / need_user_agent), then the call's own
 *     headers in the order the caller lists them (the reference iterates its HttpHeader map: for gRPC "te: trailers",
 *     "grpc-accept-encoding", "grpc-timeout" of policy/http_rpc_protocol.cpp:660-704); never-indexed when the peer announced
 *     header_table_size 0;
 *   - HEADERS (+CONTINUATION) and the body as DATA frames split at the peer's max_frame_size, END_STREAM on the last frame, the
 *     deferred connection WINDOW_UPDATE; B2_H2_REQ_GRPC prepends AddGrpcPrefix's 5 bytes (policy/http_rpc_protocol.cpp:254-262).
 * `extra` headers: records {u16 name_len, u16 value_len (little endian), name, value} back to back at extra_off, extra_len bytes.
 * On a connection opened with b2_h2_conn_reset the pending-stream count against max_concurrent_streams (:1529) and GOAWAY
 * (TryToInsertStream :425-436) belong to the caller's correlation map, and the host parses the server's frames and mirrors what they
 * change with b2_h2_conn_peer_update.  On a connection opened with b2_h2_client_conn_reset the device parses them
 * (b2_h2_client_process_batch) and this call also does what AppendAndDestroySelf does around TryToInsertStream, in its order:
 *   - pending streams > the peer's max_concurrent_streams -> B2_H2_REQ_ELIMIT, no stream id consumed (:1529-1531);
 *   - no free stream record in the connection's pool (b2_h2_configure's max_pending) -> B2_H2_REQ_NO_ROOM, no stream id consumed.
 *     This is a device capacity, not a reference error: the caller may retry after calls complete, or use another connection;
 *   - after the server's GOAWAY, a stream id above its last_stream_id -> B2_H2_REQ_LOGOFF (brpc ELOGOFF, :1559-1564), after the
 *     window was charged, as in the reference;
 *   - otherwise the stream enters the connection's pending map with the peer's stream window minus the body.
 * Requests of one connection must be adjacent and in write order. */
#define B2_H2_REQ_GRPC       1u
#define B2_H2_REQ_GET        2u     /* :method GET instead of POST */
#define B2_H2_REQ_HTTPS      4u     /* :scheme https */
#define B2_H2_REQ_ACCEPT     8u     /* need_accept: append accept: * / * */
#define B2_H2_REQ_USER_AGENT 16u    /* need_user_agent: append user-agent: brpc/1.0 curl/7.0 */
#define B2_H2_REQ_OK     0
#define B2_H2_REQ_ELIMIT 1          /* brpc ELIMIT: remote_window_left is not enough */
#define B2_H2_REQ_RUNOUT 2          /* brpc EH2RUNOUTSTREAMS */
#define B2_H2_REQ_LOGOFF 3          /* brpc ELOGOFF: the server sent GOAWAY (device-parsed client connections only) */
#define B2_H2_REQ_NO_ROOM 4         /* device capacity: the connection's stream pool is full (device-parsed client connections only) */
typedef struct b2_h2_request {
    uint32_t conn, flags;
    uint32_t path_off, path_len;                     /* inside bytes: URI::GenerateH2Path's result */
    uint32_t authority_off, authority_len;
    uint32_t content_type_off, content_type_len;     /* length 0 = no content-type header */
    uint32_t body_off, body_len;                     /* the attachment; for gRPC the serialized message */
    uint32_t extra_off, extra_len;
} b2_h2_request;                                     /* 48 bytes */
typedef struct b2_h2_request_result { int32_t status; uint32_t stream_id, out_off, out_len; } b2_h2_request_result;   /* 16 bytes */
int  b2_h2_pack_requests(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_h2_request* reqs, uint32_t n,
                         void* out, uint32_t out_cap, b2_h2_request_result* results);
/* What the peer's frames change in the state b2_h2_pack_requests / b2_h2_pack_responses read, for a connection whose frames the HOST
 * parses: H2Context::OnSettings (:848-915: _remote_settings; the first SETTINGS also takes MAX_WINDOW_SIZE - 65535 off the connection
 * window — pass it as a negative conn_window_add) and OnWindowUpdate on stream 0 (:1006-1041: AddWindowSize, B2_E_INVAL when the
 * window would pass 2^31 - 1 — FLOW_CONTROL_ERROR there).  Fields are applied when their bit is set in `set`. */
#define B2_H2_PEER_HEADER_TABLE_SIZE 1u
#define B2_H2_PEER_MAX_FRAME_SIZE    2u
#define B2_H2_PEER_STREAM_WINDOW     4u
#define B2_H2_PEER_CONN_WINDOW_ADD   8u
typedef struct b2_h2_peer_update {
    uint32_t set, header_table_size, max_frame_size, stream_window_size;
    int64_t  conn_window_add;
} b2_h2_peer_update;                                 /* 24 bytes */
int  b2_h2_conn_peer_update(b2_ctx* ctx, uint32_t conn, const b2_h2_peer_update* u);
/* the reference's own unit-test hook (:348-352: its tests start 10 000 ids before the end of the id space): the next client stream id */
int  b2_h2_conn_set_next_stream_id(b2_ctx* ctx, uint32_t conn, uint32_t next_id);

/* ---- the receiving half of an h2 / gRPC client connection, on the device --------------------------------------------------------
 * b2_h2_client_conn_reset: a new client connection whose server frames the device parses — the H2Context(socket, NULL) constructor and
 * Init (src/brpc/policy/http2_rpc_protocol.cpp:324-371): client _unack_local_settings (the flags of the preface SETTINGS that
 * b2_h2_pack_requests writes first), _local_settings until the server's ACK (equal to them at brpc's default flags), _goaway_stream_id
 * -1, fresh encoder and decoder HPACK tables.  Its stream records live in the h2 pool (b2_h2_configure).
 * b2_h2_client_process_batch: ParseH2Message on a socket created by connect, with the same arguments as b2_h2_process_batch
 * (runs = the bytes read from each client socket, runs[i].socket_id = connection, one run per connection): H2Context::Consume
 * (:467-543) looped over the run — client side: no preface is read, HEADERS / CONTINUATION for an unknown stream are still decoded
 * through the HPACK table and then dropped (:600-606, :659-665), the peer's SETTINGS / WINDOW_UPDATE update the state that
 * b2_h2_pack_requests reads (nothing to mirror).  rs[i] as there; rs[i].ctrl_off/len hold what the reference WriteAck()s, in order
 * (SETTINGS ACK, PING ACK, WINDOW_UPDATEs, RST_STREAM, GOAWAY).  A run on a connection not opened by b2_h2_client_conn_reset reads
 * nothing: B2_PARSE_ERROR_TRY_OTHERS.
 * Every stream that leaves the connection becomes one b2_h2_call, in parse order: END_STREAM (OnEndStream :825-846), the server's
 * RST_STREAM (OnResetStream :781-823, status H2ErrorToStatusCode, http2.cpp:88), a stream error of our own that sent RST_STREAM
 * (:508-528, the same status), or the server's GOAWAY (OnGoAway :959-1006 + RemoveGoAwayStreams :388-414: every pending stream above
 * last_stream_id, status 503, in ascending stream id order here — brpc's map has no order).  A GOAWAY also makes later
 * b2_h2_pack_requests on the connection refuse new streams (B2_H2_REQ_LOGOFF).
 * Each call carries what ProcessHttpResponse (policy/http_rpc_protocol.cpp:349-564) decides before it parses the response body, for
 * a call with a protobuf response type: gRPC content-type -> RemoveGrpcPrefix (ERESPONSE "Invalid gRPC response"), then a non-zero
 * grpc-status -> GrpcStatusToErrorCode (grpc.cpp:83) with the percent-decoded grpc-message or GrpcStatusToString; then :status outside
 * [200, 300) -> EHTTP "HTTP/2.0 <code> <reason>[: <first 2048 bytes of the body>]"; last, a compressed gRPC message without
 * grpc-encoding -> ERESPONSE.  error_code is the brpc errno (0: none), the text SetFailed receives is in out.  A compressed gRPC
 * message (B2_H2_FLAG_GRPC_COMPRESSED) is handed over as it is unless the connection opted in to b2_h2_conn_set_gunzip (below).
 * Header records: {u16 name_len, u16 value_len, name, value} as in b2_h2_msg, merged the way HttpHeader is filled (ConsumeHeaders
 * :1233-1288, HttpHeader::AppendHeader http_header.cpp:100-117): trailers included, pseudo-headers left out (":status" is status_code),
 * a name seen again (case-insensitive) joins the first record with "," ("; " for cookie) unless that value is empty, "content-type"
 * keeps its last value, every "set-cookie" is a record of its own; records in the order names first appear.
 * Device capacities as for the server side (b2_h2_configure), and B2_PARSE_ERROR_NO_RESOURCE ends a run whose calls or bytes do not
 * fit msg_cap / out_cap (the connection must then be closed).
 * b2_h2_client_abandon_streams: AddAbandonedStream (:1140-1143) for calls the caller gave up on (timeouts): the streams are dropped
 * where ParseH2Message runs ClearAbandonedStreams (:1103-1157) — after each frame of the next b2_h2_client_process_batch on the connection
 * that completes a call, and at the end of that run — in ascending id order here (brpc pops the most recently added first, which only
 * changes how their deferred WINDOW_UPDATE bytes are split).  So an abandoned call is still reported only if it is the first call to
 * complete in that run.  Without it their pool records stay taken. */
#define B2_H2_CALL_ENDED         0u   /* END_STREAM */
#define B2_H2_CALL_RESET_BY_PEER 1u   /* the server's RST_STREAM */
#define B2_H2_CALL_RESET_BY_US   2u   /* a stream error of ours: we sent RST_STREAM */
#define B2_H2_CALL_GOAWAY        3u   /* removed by the server's GOAWAY */
#define B2_H2_CALL_HAS_GRPC_STATUS 32u  /* flag: a grpc-status header was present */
typedef struct b2_h2_call {
    uint32_t run_idx, stream_id;
    uint32_t how;                                /* B2_H2_CALL_* */
    int32_t  status_code;                        /* :status, H2ErrorToStatusCode of a reset, 503 for GOAWAY; 200 without :status */
    int32_t  error_code;                         /* brpc errno ProcessHttpResponse sets, 0 = none */
    int32_t  grpc_status;                        /* strtol of grpc-status, -1 when absent */
    uint32_t headers_off, headers_len, n_headers;/* merged header records inside out */
    uint32_t body_off, body_len;                 /* inside out, or inside the input with B2_H2_FLAG_BODY_IN_INPUT */
    uint32_t msg_off, msg_len;                   /* gRPC message without its 5-byte prefix (B2_H2_FLAG_GRPC_PREFIX_OK), same buffer as body */
    uint32_t error_off, error_len;               /* the error text inside out */
    uint32_t flags;                              /* B2_H2_FLAG_GRPC / GRPC_PREFIX_OK / GRPC_COMPRESSED / BODY_IN_INPUT, B2_H2_CALL_HAS_GRPC_STATUS */
} b2_h2_call;                                    /* 64 bytes */
int  b2_h2_client_conn_reset(b2_ctx* ctx, uint32_t conn);
int  b2_h2_client_process_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                                b2_h2_run_status* rs, b2_h2_call* calls, uint32_t call_cap, uint32_t* n_calls,
                                void* out, uint32_t out_cap);
int  b2_h2_client_abandon_streams(b2_ctx* ctx, uint32_t conn, const uint32_t* stream_ids, uint32_t n);

/* ---- gzip-compressed h2 / gRPC messages, inflated on the device (opt-in per connection) ------------------------------------------
 * b2_h2_conn_set_gunzip: the connection's messages are protobuf-typed, so the next b2_h2_process_batch (server connections) or
 * b2_h2_client_process_batch (device-parsed client connections) also does what ProcessHttpRequest (policy/http_rpc_protocol.cpp:
 * 1645-1683) / ProcessHttpResponse (:507-529) do before the protobuf parse:
 *   - the encoding: gRPC content-type -> the merged "grpc-encoding" value, only when the prefix's compressed flag is set (a message
 *     sent uncompressed with "grpc-encoding: gzip", as grpc clients and servers send small ones, is left alone); other messages ->
 *     the merged "content-encoding" value.  It must be exactly "gzip" (case and all; "gzip" sent twice merges into "gzip,gzip");
 *   - candidates: server messages with a valid gRPC prefix or, not gRPC, a non-empty body; client calls with error_code 0 (so a call
 *     with an invalid prefix, a non-zero grpc-status or a non-2xx status is never inflated);
 *   - policy::GzipDecompress: GzipInputStream(GZIP) over the message as ONE block (as the baidu_std gzip bodies), which cannot fail;
 *     a damaged stream yields what zlib handed over before the error.  brpc reads a body of several IOBuf blocks and can then answer
 *     "Fail to un-gzip ..." depending on where the blocks end; the device never does.
 * The inflated bytes land in out, 16-byte aligned after what the parse itself wrote in the run's region, in message order; a
 * message whose size bound does not fit there is skipped (B2_H2_FLAG_GUNZIP_HOST) and later ones are still tried.  A server message
 * echoed from there needs no copy: b2_h2_pack_responses with B2_H2_RESP_BODY_IN_OUT.  b2_h2_conn_reset and b2_h2_client_conn_reset
 * clear the setting; batches without such a connection run exactly as before. */
#define B2_H2_FLAG_GUNZIPPED        64u   /* inflated: msg_off/msg_len index the inflated bytes in out (body_* still the received body) */
#define B2_H2_FLAG_GUNZIP_HOST     128u   /* would be inflated, left as received: > 1 MiB compressed or inflated, or no room in out */
#define B2_H2_FLAG_NO_GRPC_ENCODING 256u  /* compressed gRPC message without grpc-encoding (brpc: EREQUEST / ERESPONSE "Fail to find header");
                                             not set on a client call an earlier verdict already failed */
int  b2_h2_conn_set_gunzip(b2_ctx* ctx, uint32_t conn, int enable);

/* ---- gRPC calls to device echo methods answered on the device, in the parse call ------------------------------------------------
 * b2_h2_serve_batch: b2_h2_process_batch, then for the calls it can answer what brpc does next — ProcessHttpRequest's body checks
 * (policy/http_rpc_protocol.cpp:1631-1689), EchoServiceImpl::Echo, SendHttpResponse (:852-1027) — framed like b2_h2_pack_responses.
 * rs, msgs and out are what b2_h2_process_batch returns for the same input (gunzip included), except that answered calls carry
 * B2_H2_FLAG_ANSWERED and their reply's grpc-status in msgs[i].reserved.
 * A call is answered when it is gRPC, its content type is HTTP_CONTENT_PROTO, method_idx names a B2_HANDLER_ECHO method whose
 * response_compress_type is NONE, and its content-type value is at most 256 bytes; everything else (unknown paths included) is left to
 * the host unchanged.  The verdicts, in the reference's order, each an EREQUEST reply unless the call is OK:
 *   - an empty body: "<request_type_name> needs to be created from a non-empty json, it has required fields." (:1637-1643);
 *   - RemoveGrpcPrefix fails: "Invalid gRPC request";
 *   - a compressed message with B2_H2_FLAG_NO_GRPC_ENCODING: "Fail to find header `grpc-encoding' in compressed gRPC request";
 *     with B2_H2_FLAG_GUNZIPPED the inflated bytes go on; any other compressed message is not answered;
 *   - the message is not an EchoRequest (proto2, required `message`): "Fail to parse http body as <request_type_name>";
 *   - OK: :status 200, the request's content-type, the body EchoResponse{message} (0a varint(len) message: referenced in the input or
 *     the inflated bytes when the request holds exactly those bytes, else written into the run's out region), grpc-status 0.
 * An error reply is :status 200, the request's content-type, an empty message (5-byte prefix), grpc-status 3 (ErrorCodeToGrpcStatus,
 * grpc.cpp:54-81) and grpc-message = PercentEncode (grpc.cpp:121-141: a-z A-Z - _ . ~ kept, every other byte "%xx") of the text
 * Controller::SetFailed builds (controller.cpp:468-490): "[ip:port]" (b2_set_server_identity, when set), "[E1003]", the reason.  Up to 702
 * bytes; the text is written into the run's out region.  A call whose bytes do not fit behind the parse's and the gunzip's bytes in the
 * run's out region is not answered; later calls still may be.
 * Replies: run i's region of `replies` is replies_cap / n_runs bytes (rounded down to 64).  Each answered call reserves the bound of
 * b2_h2_pack_responses there; when the next does not fit, the run's remaining calls are not answered.  Run i's replies are
 * replies[spans[i].off, + spans[i].len), in message order, spans[i].n_answered of them: write them after rs[i].ctrl_*.  The encoder
 * HPACK table, the remote windows and the deferred WINDOW_UPDATE end as after b2_h2_process_batch + b2_h2_pack_responses on the same
 * records, and the call leaves the batch readable by b2_h2_pack_responses: the host answers the rest, zero-copy as before.
 * replies_cap <= the context's max_resp_bytes.  Not modelled: concurrency limiters (EOVERCROWDED), auth, grpc-timeout; a request
 * attachment is always empty here, so echo_attachment changes nothing. */
#define B2_H2_FLAG_ANSWERED 512u   /* b2_h2_msg.flags: the device wrote this call's reply (b2_h2_serve_batch) */
typedef struct b2_h2_reply_span { uint32_t off, len, n_answered, reserved; } b2_h2_reply_span;   /* 16 bytes */
int  b2_h2_serve_batch(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                       b2_h2_run_status* rs, b2_h2_msg* msgs, uint32_t msg_cap, uint32_t* n_msgs, void* out, uint32_t out_cap,
                       void* replies, uint32_t replies_cap, b2_h2_reply_span* spans);
/* h2/gRPC on the latency path: b2_h2_serve_batch inside a resident kernel (k_h2_ring) fed through the submit ring of b2_ring_* — no
 * launch, copy or stream synchronisation per batch.  A context runs either k_ring or k_h2_ring, never both: its first ring call (an enable
 * call, b2_ring_start or b2_ring_submit) fixes which resident kernel it runs.
 * b2_h2_ring_enable: once, after b2_h2_configure and before the context's first ring call (after b2_ring_start / b2_ring_submit /
 * b2_stream_ring_enable, or twice: B2_E_INVAL; b2_ring_submit / b2_ring_wait then fail with B2_E_INVAL).  The four capacities are per
 * ticket and play the roles of b2_h2_serve_batch's nbytes bound, msg_cap, out_cap and replies_cap; they are checked against the context
 * limits that call checks and fix the slot layout (header, runs, staged input, statuses, messages, spans, out, replies, times the 8 ring
 * slots, all pinned + mapped host memory).  b2_ring_stop, b2_ring_launches, b2_ring_phase_ns ([2]: replies packed) and
 * B2_RING_IDLE_MS apply to k_h2_ring as to k_ring.
 * b2_h2_ring_submit: the argument checks of b2_h2_serve_batch (runs inside the buffer, socket_id < max_conns, one run per connection,
 * n_runs <= max_runs, (out_cap / n_runs) & ~63 >= 256 and msg_cap / n_runs > 0), n_runs > 0, and nbytes <= max_bytes (else
 * B2_E_CAPACITY: serve that batch with b2_h2_serve_batch).  Bytes in b2_block_alloc memory are pulled in place, others staged into the
 * slot.  Connections with gunzip on (b2_h2_conn_set_gunzip) are served too.
 * b2_h2_ring_wait: tickets may be waited in any order.  For any sequence of tickets the results equal, byte for byte, what
 * b2_h2_serve_batch returns for the same sequence of batches with the same caps: run statuses, messages (B2_H2_FLAG_ANSWERED, the
 * grpc-status in `reserved`), the defined bytes of out (run i's control bytes at ctrl_off, its blob from i * region + region / 4),
 * spans and replies — and so does the connection state left behind (HPACK tables, windows, deferred WINDOW_UPDATEs, the stream pool).
 * After the wait of the most recent ticket, b2_h2_pack_responses resolves B2_H2_RESP_BODY_IN_INPUT / _BODY_IN_OUT / _CT_IN_OUT
 * against that ticket, as after the batch call.
 * While a ticket is outstanding every call that uploads to the context or touches h2 state fails with B2_E_INVAL: the b2_h2_* and
 * b2_hpack_* calls, the batch calls (b2_batch_upload / _submit, b2_process_batch), b2_pack_*, b2_crc32c_batch, the snappy batch calls,
 * b2_stream_write and b2_set_server_identity — the ticket uses their device scratch.  Between tickets every call is allowed.  A call that
 * writes h2 connection state (b2_h2_conn_reset / _set_gunzip / _peer_update / _set_next_stream_id, b2_h2_client_*, b2_h2_process_batch,
 * b2_h2_serve_batch, b2_h2_pack_*, b2_hpack_*) and b2_set_server_identity first retire the resident kernel, which reads that state
 * through L1; the next submission relaunches it (b2_ring_launches counts it). */
typedef struct b2_h2_ring_result {    /* views into the ticket's pinned slot, valid until the slot is reused by the 8th later submission */
    const b2_h2_run_status* runs; uint32_t n_runs, n_msgs;
    const b2_h2_msg* msgs;            /* compacted: runs[i].first_msg is a list index, as b2_h2_serve_batch returns it */
    const uint8_t* out; uint32_t region;   /* run i's control bytes and blob live at out + i * region, as in the batch call */
    const uint8_t* replies; const b2_h2_reply_span* spans;
    int32_t status;                   /* what b2_h2_serve_batch would have returned for this batch */
} b2_h2_ring_result;                  /* 64 bytes */
int  b2_h2_ring_enable(b2_ctx* ctx, uint32_t max_bytes, uint32_t msg_cap, uint32_t out_cap, uint32_t replies_cap);
int  b2_h2_ring_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs, uint32_t* ticket);
int  b2_h2_ring_wait(b2_ctx* ctx, uint32_t ticket, b2_h2_ring_result* out);
/* A gRPC server's TURN on the latency path: one ticket of k_h2_ring that serves what arrived, exactly as b2_h2_serve_batch, and then sends
 * the replies user code produced for earlier calls, exactly as b2_h2_pack_responses — with no relaunch, launch, copy or stream
 * synchronisation for the host's replies.  (b2_h2_pack_responses between tickets still works, and still retires the resident kernel.)
 * Inside a turn the order is read, then write: a SETTINGS or WINDOW_UPDATE in the runs governs how that turn's host replies are framed and
 * charged (max_frame_size, header_table_size 0 = never-indexed, a connection window that no longer covers a body gives
 * RST_STREAM(FLOW_CONTROL_ERROR)), and the turn's device-answered replies take the HPACK encoder before the host's.  Per connection write
 * its run's control bytes (ctrl_off / ctrl_len), then its device replies (spans[i]), then its host replies in record order.
 * b2_h2_ring_turn_enable: everything b2_h2_ring_enable does, with the same rules and caps; max_resps and resp_out_cap are per turn and play
 * the roles of b2_h2_pack_responses' n and out_cap (max_resps <= max_msgs, resp_out_cap and max_bytes <= max_resp_bytes, else
 * B2_E_CAPACITY).  They add the host-reply parts to each slot and device scratch of their own.
 * b2_h2_ring_turn_submit: the checks of b2_h2_ring_submit when n_runs > 0, then every check of b2_h2_pack_responses on the replies with the
 * turn's caps: the connection in range, replies of one connection adjacent, fields inside `bytes`, content-type <= 256 and grpc-message
 * <= 512 bytes (B2_E_INVAL), n_resps <= max_resps and room by h2_reply_bound within resp_out_cap (B2_E_CAPACITY).  The records are
 * b2_h2_response, unchanged; their fields index the turn's own bytes, the same buffer as the runs.  B2_H2_RESP_BODY_IN_INPUT,
 * _BODY_IN_OUT and _CT_IN_OUT are refused (B2_E_INVAL): they name the previous ticket's device buffers, which this ticket's pull
 * overwrites.  A turn carries runs, replies or both, not neither (B2_E_INVAL); a reply-only turn sends replies without waiting for the next
 * read.
 * b2_h2_ring_turn_wait: tickets may be waited in any order.  For any sequence of turns the results equal, byte for byte, what a context
 * returns for the same sequence of b2_h2_serve_batch(bytes, runs, ...) + b2_h2_pack_responses(bytes, resps, ...) with the same caps (a
 * call whose list is empty skipped): `ring` as b2_h2_ring_wait fills it (ring.status B2_E_CAPACITY when the served half would fail; the
 * host replies are packed all the same, as the two calls in a row would), each reply's frame bytes and length — and so does the
 * connection state left behind (both HPACK tables, the windows, the deferred WINDOW_UPDATE, the stream pool).  After the wait of the most
 * recent ticket, b2_h2_pack_responses resolves the zero-copy flags against it as after b2_h2_ring_wait.
 * On a turn-enabled context b2_h2_ring_submit / _wait still serve tickets without replies; the turn calls on a b2_h2_ring_enable context
 * fail with B2_E_INVAL.  Every refusal and retirement rule of b2_h2_ring_wait above applies.  Compressed replies stay with the batch calls. */
typedef struct b2_h2_ring_turn_result {  /* views into the ticket's pinned slot, valid until the slot is reused by the 8th later submission */
    b2_h2_ring_result ring;              /* the served half, as b2_h2_ring_wait returns it */
    uint32_t n_resps, reserved;
    const uint32_t* resp_offs;           /* host reply i: resp_out[resp_offs[i], + resp_lens[i]) */
    const uint32_t* resp_lens;
    const uint8_t* resp_out;
} b2_h2_ring_turn_result;                /* 96 bytes */
int  b2_h2_ring_turn_enable(b2_ctx* ctx, uint32_t max_bytes, uint32_t msg_cap, uint32_t out_cap, uint32_t replies_cap,
                            uint32_t max_resps, uint32_t resp_out_cap);
int  b2_h2_ring_turn_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                            const b2_h2_response* resps, uint32_t n_resps, uint32_t* ticket);
int  b2_h2_ring_turn_wait(b2_ctx* ctx, uint32_t ticket, b2_h2_ring_turn_result* out);
/* h2/gRPC CLIENT connections on the latency path: b2_h2_client_process_batch followed by b2_h2_pack_requests inside a resident kernel
 * (k_h2_client_ring) fed through the same submit ring.  A ticket is one turn of a client's event loop: read what arrived, then send what
 * is queued.  The runs (the bytes read from client sockets, socket_id = connection) are parsed as by b2_h2_client_process_batch, then the
 * requests are packed as by b2_h2_pack_requests; their fields index the same `bytes` as the runs.  So within one ticket a SETTINGS or
 * WINDOW_UPDATE in the runs governs how its requests are framed and charged, a GOAWAY in the runs makes its later stream ids
 * B2_H2_REQ_LOGOFF, and calls that end in the runs free their stream records before the requests take records (B2_H2_REQ_NO_ROOM).
 * For each connection write its run's control bytes (ctrl_off / ctrl_len) first, then its request frames in request order.
 * A context runs exactly one of k_ring, k_h2_ring and k_h2_client_ring: b2_ring_submit / _wait, b2_h2_ring_* and b2_stream_ring_enable
 * refuse a context that runs this one, and b2_h2_client_ring_enable refuses a context that ran another.
 * b2_h2_client_ring_enable: once, after b2_h2_configure and before the context's first ring call (else B2_E_INVAL).  The caps are per
 * ticket and play the roles of the batch calls' nbytes bound (both), call_cap and out_cap (b2_h2_client_process_batch), and the number
 * of requests and out_cap (b2_h2_pack_requests); they are checked against the context limits those calls check and fix the slot layout.
 * b2_ring_stop, b2_ring_launches, b2_ring_phase_ns ([2]: requests packed) and B2_RING_IDLE_MS apply as to k_h2_ring.
 * b2_h2_client_ring_submit: every check of both batch calls with the enable-time caps; n_runs or n_reqs may be 0, not both.  Bytes in
 * b2_block_alloc memory are pulled in place, others staged into the slot.
 * b2_h2_client_ring_wait: tickets may be waited in any order.  For any sequence of tickets the results equal, byte for byte, what a context
 * returns for the same sequence of b2_h2_client_process_batch(bytes, runs, call_cap, out_cap) + b2_h2_pack_requests(bytes, reqs,
 * req_out_cap) (a call whose list is empty skipped): run statuses and calls, the defined bytes of out, request results and each request's
 * frames — and so does the connection state left behind (HPACK tables, windows, deferred WINDOW_UPDATEs, the pending map, stream ids,
 * GOAWAY).  A client ticket leaves nothing for b2_h2_pack_responses to read zero-copy, as the client batch call.
 * While a ticket is outstanding the calls b2_h2_ring_wait lists above fail with B2_E_INVAL, and the calls that write h2 connection state
 * (b2_h2_client_conn_reset / _abandon_streams, b2_h2_conn_set_gunzip / _peer_update / _set_next_stream_id, ...) retire the kernel between
 * tickets; the next submission relaunches it (b2_ring_launches counts it). */
typedef struct b2_h2_client_ring_result {       /* views into the ticket's pinned slot, valid until the 8th later submission */
    const b2_h2_run_status* runs; uint32_t n_runs, n_calls;
    const b2_h2_call* calls;                    /* compacted: runs[i].first_msg is a list index */
    const uint8_t* out; uint32_t region;        /* run i's control bytes and blob at out + i * region, as in the batch call */
    uint32_t n_reqs;
    const b2_h2_request_result* reqs;           /* status, stream_id, out_off, out_len */
    const uint8_t* req_out;                     /* request i's frames at req_out + reqs[i].out_off */
    int32_t status; uint32_t reserved;
} b2_h2_client_ring_result;                     /* 64 bytes */
int  b2_h2_client_ring_enable(b2_ctx* ctx, uint32_t max_bytes, uint32_t call_cap, uint32_t out_cap, uint32_t max_reqs, uint32_t req_out_cap);
int  b2_h2_client_ring_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                              const b2_h2_request* reqs, uint32_t n_reqs, uint32_t* ticket);
int  b2_h2_client_ring_wait(b2_ctx* ctx, uint32_t ticket, b2_h2_client_ring_result* out);

/* ---- streaming_rpc, the receiving side of a Stream on the device ------------------------------------------------------------------
 * Without a stream table a STRM frame ends as a B2_MSG_STREAM_FRAME descriptor and the host rebuilds brpc's Stream from the list.  With
 * one (b2_stream_configure) every batch call also runs, behind the stage that writes msgs[] and inside the same synchronisation, what
 * brpc does per frame after the meta parse:
 *   ParseStreamingMessage (src/brpc/policy/streaming_rpc_protocol.cpp:99-129): the id is looked up; a frame for an id that is not open
 *     (never opened, closed in an earlier batch or earlier in this one) is answered with SendStreamRst (:139-149) when it carries a
 *     source_stream_id and is not a FEEDBACK, and does nothing else;
 *   Stream::OnReceived (src/brpc/stream.cpp:499-543): DATA payloads are appended until a frame whose has_continuation VALUE is false
 *     completes the message; FEEDBACK -> remote_consumed = max(remote_consumed, consumed_size) (SetRemoteConsumed :362-401, with
 *     -socket_max_streams_unconsumed_bytes at its default 0); RST -> closed with ECONNRESET, CLOSE -> closed with 0 (Close :710-732),
 *     the partial message is dropped; any other frame_type is ignored;
 *   Stream::Consume (:582-651) + SendFeedback (:653-662), ONCE per stream per batch: local_consumed += the bytes of the messages the
 *     batch completed, and when that is > 0 on a CONNECTED stream whose peer set need_feedback one FEEDBACK frame with the cumulative
 *     count; BeforeRecycle (:129-146): the CLOSE frame of a connected stream that was closed.
 * Decisions brpc leaves to bthread scheduling: one Consume per stream per batch; a stream closed in a batch still delivers the messages
 * completed before the close and writes FEEDBACK before CLOSE; frames of one stream are ordered by their msgs[] index, whichever
 * socket they came in on.  The per-frame b2_msg_desc records stay exactly as without a table (B2_STREAM_SNAPPY_UNCOMPRESS included).
 * Capacity (the reference has none): a partial message that outgrows pending_bytes, or a multi-frame message that no longer fits the
 * out region of the batch, puts the stream into HANDED_OVER — the event names the first descriptor the device did not absorb
 * (handover_msg), the parts gathered in earlier batches are fetched once with b2_stream_take_pending, and from then on the stream's
 * frames are described per frame only (no routing, no RST) until b2_stream_close.
 * Not modelled: _parse_rpc_response (open a client stream after the host took the RPC response), idle timers, messages_in_batch.
 * The ring path runs the pass only after b2_stream_ring_enable (below); without it b2_ring_submit fails with B2_E_INVAL on a context
 * that has a table.  The measurement entry
 * points (b2_batch_execute, b2_batch_execute_many, b2_batch_launch) do not run it either: they replay one batch, and fail with
 * B2_E_INVAL between b2_batch_submit and b2_batch_collect on a context with a table.  When one batch completes more multi-frame bytes
 * than the out region holds, WHICH of the competing streams is handed over is unspecified (room is handed out as the warps ask). */
#define B2_STREAM_CONNECTED      1u   /* b2_stream_desc.flags: Stream::_connected, remote_stream_id is valid */
#define B2_STREAM_NEED_FEEDBACK  2u   /* _remote_settings.need_feedback */
#define B2_STREAM_CLOSED         4u   /* b2_stream_state.flags */
#define B2_STREAM_HANDED_OVER    8u
typedef struct b2_stream_desc {
    int64_t  stream_id;               /* what peers put in StreamFrameMeta.stream_id */
    int64_t  remote_stream_id;        /* _remote_settings.stream_id (CONNECTED) */
    uint64_t host_socket_id;          /* opaque; echoed in the events: where FEEDBACK / CLOSE go */
    uint32_t flags;
    uint32_t max_buf_size;            /* StreamOptions::max_buf_size when > 0: the write window (b2_stream_write); 0 = no window */
} b2_stream_desc;                     /* 32 bytes */
typedef struct b2_stream_state {
    uint64_t local_consumed, remote_consumed;
    uint32_t pending_bytes;           /* bytes of the partial message that waits on the device */
    uint32_t flags;                   /* B2_STREAM_* */
    int32_t  error_code;              /* of the close: ECONNRESET (104) after RST, 0 after CLOSE */
    uint32_t reserved;
} b2_stream_state;                    /* 32 bytes */
#define B2_STREAM_MSG_IN_INPUT 1u     /* off indexes the request bytes (one frame carried the message: zero copy), else the out region */
typedef struct b2_stream_msg {
    int64_t  stream_id;
    uint32_t first_frame;             /* b2_msg_desc index of the message's first frame in THIS batch */
    uint32_t n_frames;                /* DATA frames of the message, earlier batches included */
    uint32_t off, len;
    uint32_t flags, reserved;
} b2_stream_msg;                      /* 32 bytes */
#define B2_STREAM_EV_REMOTE_CONSUMED_MOVED 1u
#define B2_STREAM_EV_CLOSED_BY_RST         2u   /* error ECONNRESET */
#define B2_STREAM_EV_CLOSED_BY_CLOSE       4u   /* error 0 */
#define B2_STREAM_EV_HANDED_OVER           8u
#define B2_STREAM_EV_WRITABLE             16u   /* a FEEDBACK of this batch took the stream from full to not full: wake StreamWait */
typedef struct b2_stream_event {
    int64_t  stream_id;
    uint64_t host_socket_id;
    uint64_t local_consumed, remote_consumed;   /* after the batch */
    uint32_t n_msgs, first_msg;       /* the stream's completed messages: b2_stream_batch_result.msgs[first_msg, +n_msgs), arrival order */
    uint32_t consumed_bytes;          /* of this batch */
    uint32_t flags;                   /* B2_STREAM_EV_* */
    uint32_t fb_off, fb_len;          /* FEEDBACK frame inside ctrl (len 0 = none) */
    uint32_t close_off, close_len;    /* CLOSE frame inside ctrl, to be written after the FEEDBACK */
    uint32_t handover_msg;            /* HANDED_OVER: first b2_msg_desc of the stream the device did not absorb */
    uint32_t pending_bytes;           /* bytes of the partial message kept on the device after the batch */
    uint32_t reserved[2];
} b2_stream_event;                    /* 80 bytes */
/* Pointers into ctx-owned pinned memory, valid after b2_process_batch / b2_batch_collect until the next batch call on the context.
 * msgs are grouped by stream; the order of streams (and of the spans inside out / ctrl) is not specified. */
typedef struct b2_stream_batch_result {
    const b2_stream_msg*   msgs;    uint32_t n_msgs;
    const b2_stream_event* events;  uint32_t n_events;     /* one per stream the batch touched */
    const uint8_t*         out;     uint32_t out_bytes;    /* reassembled multi-frame messages */
    const uint8_t*         ctrl;    uint32_t ctrl_bytes;   /* wire-ready frames to write */
    const uint32_t*        run_ctrl; uint32_t n_runs;      /* [2 * n_runs] {off, len} inside ctrl: run i's RST frames, in message order,
                                                              to be written to the socket the run came from */
} b2_stream_batch_result;
/* Before the first batch call.  max_streams open streams; pending_bytes (multiple of 16) per stream for a message that spans batches;
 * out_bytes for the multi-frame messages one batch completes (0 = the context's max_batch_bytes). */
int  b2_stream_configure(b2_ctx* ctx, uint32_t max_streams, uint32_t pending_bytes, uint32_t out_bytes);
/* StreamAccept / StreamCreate: the ids start resolving.  Between batch calls. */
int  b2_stream_open(b2_ctx* ctx, const b2_stream_desc* streams, uint32_t n);
/* Stream::SetConnected(remote_settings) of a client-side stream whose settings arrive with the RPC response (stream.cpp:270-307):
 * flags = B2_STREAM_NEED_FEEDBACK or 0.  frame / frame_len: its first FEEDBACK when bytes were consumed before (frame_cap >= 64). */
int  b2_stream_set_connected(b2_ctx* ctx, int64_t stream_id, int64_t remote_stream_id, uint32_t flags, void* frame, uint32_t frame_cap, uint32_t* frame_len);
/* Local close: the id stops resolving and its table slot is free again.  frame / frame_len: the CLOSE frame when the stream was
 * connected and the peer had not closed it (frame_cap >= 64). */
int  b2_stream_close(b2_ctx* ctx, int64_t stream_id, void* frame, uint32_t frame_cap, uint32_t* frame_len);
int  b2_stream_query(b2_ctx* ctx, int64_t stream_id, b2_stream_state* out);
/* The partial message of a stream (a HANDED_OVER one hands it out this way), at most cap bytes; it is gone from the device afterwards. */
int  b2_stream_take_pending(b2_ctx* ctx, int64_t stream_id, void* out, uint32_t cap, uint32_t* len);
int  b2_stream_results(b2_ctx* ctx, b2_stream_batch_result* out);
/* The stream pass on the latency path: after b2_stream_configure and before the context's first ring call (later, or twice:
 * B2_E_INVAL).  k_ring then runs the pass of every ticket on the same table, with the same rules and results as a batch call.
 * out_bytes: the reassembled multi-frame bytes one ticket may complete (a ticket that completes more hands streams over by the rule
 * above; the batch calls keep b2_stream_configure's out region).  After b2_ring_wait(t), b2_stream_results describes ticket t: pointers
 * into the slot's stream section, valid until the slot is reused by the 8th later submission (or, for a ticket that overflowed the
 * compact block, the batch call's results, valid until the next call).  While a ticket is outstanding, b2_stream_open / _set_connected /
 * _close / _take_pending and b2_stream_write fail with B2_E_INVAL and leave the table untouched; between tickets they work as always.
 * B2_STREAM_W_FROM_MSG after ring tickets resolves against the ticket b2_stream_results describes, and only while that is the most
 * recent ticket: its B2_STREAM_MSG_IN_INPUT messages are read from the ring's device copy of its input and its out-region messages from
 * the ring's device out region, both overwritten by the next ticket; otherwise every FROM_MSG index fails with B2_E_INVAL.  The table,
 * the pool and the pending messages live in device memory and survive the kernel's idle retirement and relaunch unchanged. */
int  b2_stream_ring_enable(b2_ctx* ctx, uint32_t out_bytes);

/* ---- streaming_rpc, the sending side of a Stream on the device ---------------------------------------------------------------------
 * b2_stream_write: brpc::StreamWrite (src/brpc/stream.cpp:782-794) for a batch of writes against the stream table, applied in array
 * order as if one thread called StreamWrite for each in turn.  Per write, in this order:
 *   Socket::Address (:785-788): an id that is not open — never opened, closed locally, or closed by the peer's RST / CLOSE (Close
 *     SetFailed's the fake socket, :710) — gets EINVAL (produced and host_socket_id 0);
 *   a HANDED_OVER stream gets B2_STREAM_W_HANDED_OVER: its FEEDBACK frames reach only the host, so the device window is stale;
 *   AppendIfNotFull (:326-360): with max_buf_size > 0 and produced >= remote_consumed + max_buf_size -> EAGAIN, nothing charged; else
 *     produced += len (checked BEFORE the add, so one write may overshoot the window).  Without a window produced is not kept (0);
 *   Socket::Write of an empty message (socket.cpp:1609-1610) -> EINVAL (after the window check, produced -= 0);
 *   a stream that is not connected -> B2_STREAM_W_NOT_CONNECTED, nothing charged (brpc queues such writes in the fake socket until
 *     SetConnected; the device has no remote_stream_id to frame them with: write again after b2_stream_set_connected);
 *   else the frames (CutMessageIntoFileDescriptor :148-215 + PackStreamMessage, policy/streaming_rpc_protocol.cpp:42-58): "STRM",
 *     BE32 body_size, BE32 meta_size, StreamFrameMeta{stream_id = remote_stream_id, source_stream_id = id, frame_type = DATA,
 *     has_continuation}, the payload.  len > max_segment_size is cut into ceil(len / seg) frames, all but the last with
 *     has_continuation = true; otherwise one frame with has_continuation = false.
 * Each admitted write's frames are contiguous at out + results[i].out_off; out_off is 16-aligned and grows in array order, and the
 * alignment gaps between writes are zero bytes.  Write them to
 * host_socket_id in array order (WriteToHostSocket).  brpc leaves the interleaving of different streams on one socket to scheduling;
 * this call fixes it to array order.  Not modelled: _remote_settings.writable() (brpc fails such writes later with EBADF: check it
 * before writing), window adaptation (-socket_max_streams_unconsumed_bytes / min_buf_size), write_in_background, StreamWait timeouts.
 * The call checks everything before any state changes and then fails with B2_E_INVAL / B2_E_CAPACITY: no table, a batch submitted and
 * not collected, an unknown flag, src_off + src_len > nbytes, a FROM_MSG index not below the last collected batch's n_msgs, more
 * writes than max_msgs, nbytes > max_batch_bytes, or out_cap (and max_resp_bytes) below the sum over writes of
 * align16(len + ceil(len / seg) * 38) (38: the longest DATA frame head, 12 + a 26-byte meta; len 0 counts as one frame).
 * B2_STREAM_W_FROM_MSG takes the payload where the receive pass left msgs[src_off] of the last collected batch (b2_stream_results):
 * the batch's input bytes (B2_STREAM_MSG_IN_INPUT: the device copy, or the caller's mapped region with B2_INPUT_PULL, which must be
 * unchanged) or the stream out region — nothing crosses PCIe to the device.  The device copy of the batch's input lasts until the next
 * call that uploads bytes to the context (b2_pack_*, b2_h2_*, b2_hpack_decode_batch, b2_crc32c_batch, the snappy batch calls; a batch
 * call ends the last batch altogether): after such a call a FROM_MSG write of a B2_STREAM_MSG_IN_INPUT message fails with B2_E_INVAL,
 * while out-region messages (and, with B2_INPUT_PULL, the caller's region) can still be written.
 * The call has its own staging: b2_stream_results and b2_batch_result stay valid and unchanged across any number of write calls. */
#define B2_STREAM_W_FROM_MSG       1u    /* payload = msgs[src_off] of the last collected batch's b2_stream_batch_result */
#define B2_STREAM_W_NOT_CONNECTED  (-1)  /* statuses of the device; negative, so they never collide with an errno */
#define B2_STREAM_W_HANDED_OVER    (-2)
typedef struct b2_stream_write_desc {
    int64_t  stream_id;               /* the local StreamId (b2_stream_desc.stream_id) */
    uint32_t flags;                   /* B2_STREAM_W_FROM_MSG */
    uint32_t src_off, src_len;        /* the message inside `bytes`; FROM_MSG: src_off = message index, src_len ignored */
    uint32_t reserved;
} b2_stream_write_desc;               /* 24 bytes (not "b2_stream_write": that name is the function) */
typedef struct b2_stream_write_result {
    int32_t  status;                  /* what StreamWrite returns: 0, EAGAIN, EINVAL; or B2_STREAM_W_* */
    uint32_t n_frames;
    uint32_t out_off, out_len;        /* the write's frames inside out (len 0 unless status 0) */
    uint64_t produced;                /* _produced after this write */
    uint64_t host_socket_id;          /* where the frames go (WriteToHostSocket) */
} b2_stream_write_result;             /* 32 bytes */
/* max_segment_size: -stream_write_max_segment_size (stream.cpp:39); 0 = brpc's default, 512 MiB. */
int  b2_stream_write(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_stream_write_desc* writes, uint32_t n,
                     uint32_t max_segment_size, void* out, uint32_t out_cap, b2_stream_write_result* results);
/* A Stream producer's turn on the latency path: b2_process_batch followed by b2_stream_write inside the resident k_ring
 * (k_ring<RingBody::stream_writes>) fed through the same submit ring.  A ticket is one turn: read the FEEDBACK / RST / CLOSE (and DATA)
 * frames the peers sent, then write what is queued.  Its runs are served as b2_ring_submit serves them on a context with
 * b2_stream_ring_enable (the batch, then the stream pass); then its writes are applied as b2_stream_write applies them, in array order,
 * against the table the stream pass just updated.  brpc leaves the race between a socket's read and StreamWrite callers to scheduling;
 * here a ticket reads first: a FEEDBACK in its runs moves remote_consumed before its writes are admitted, and an RST / CLOSE in its runs
 * closes the stream before its writes (EINVAL).  B2_STREAM_EV_WRITABLE keeps its meaning: produced does not move during the stream pass.
 * A context runs one ring kind: b2_ring_submit / _wait and the other kinds' calls refuse a context that runs this one, and
 * b2_stream_ring_* refuse a context of another kind.  Every rule of b2_stream_ring_enable holds: tickets are collected in ticket order,
 * the table calls and b2_stream_write fail with B2_E_INVAL while a ticket is outstanding, and b2_stream_results describes the ticket
 * after its wait (an empty pass for a ticket without runs).
 * b2_stream_ring_write_enable: after b2_stream_ring_enable and before the context's first ring call (else B2_E_INVAL).  max_bytes bounds
 * a ticket's whole `bytes` (the runs' bytes plus the write payloads, <= max_batch_bytes, so a turn may exceed b2_ring_submit's 128 KiB);
 * max_writes (<= max_msgs) and write_out_cap (<= max_resp_bytes) play the roles of b2_stream_write's n and out_cap; max_segment_size has
 * b2_stream_write's meaning (0 = 512 MiB) for every ticket.  Caps above those limits fail with B2_E_CAPACITY; they fix the slot layout.
 * b2_ring_stop, b2_ring_launches, b2_ring_phase_ns ([2]: runs, stream pass and writes done) and B2_RING_IDLE_MS apply as to k_ring.
 * b2_stream_ring_submit: n_runs or n_writes may be 0, not both.  Every check of b2_ring_submit (<= 512 runs, 16-aligned runs inside
 * `bytes`) and of b2_stream_write (n_writes <= max_writes, known flags, payloads inside `bytes`, the sum over writes of
 * align16(len + ceil(len / seg) * 38) <= write_out_cap: B2_E_CAPACITY) applies with the enable-time caps; a failed check claims no slot
 * and leaves the next ticket number unchanged.  Write payloads index the same `bytes` as the runs.  B2_STREAM_W_FROM_MSG is refused
 * (B2_E_INVAL): which messages a ticket completes is not known when it is submitted; echo a received message with b2_stream_write
 * between tickets, which resolves FROM_MSG against the most recent ticket.  The runs keep the compact block's limits, sized from the extent
 * the runs cover.  Bytes in b2_block_alloc memory are pulled in place, others staged into the slot.
 * b2_stream_ring_wait: for any sequence of tickets, `batch`, b2_stream_results, every write result and the frames (the zero gaps between
 * writes included, out_bytes of them) equal, byte for byte, what a context with the same table returns for b2_process_batch(bytes, runs)
 * followed by b2_stream_write(bytes, writes, max_segment_size), each call skipped when its list is empty; so does b2_stream_query of every
 * stream afterwards.  A ticket whose runs overflow the compact block has its runs served through the big pipeline inside the wait, then
 * its writes through b2_stream_write's kernels, and only then does the kernel serve the next ticket.  `bytes` must stay unchanged until
 * the ticket is collected. */
typedef struct b2_stream_ring_result {      /* views into the ticket's pinned slot, valid until the 8th later submission */
    b2_batch_result batch;                  /* the runs, exactly as b2_ring_wait returns them */
    uint32_t n_writes, out_bytes;
    const b2_stream_write_result* results;  /* as b2_stream_write's results */
    const uint8_t* out;                     /* write i's frames at out + results[i].out_off */
} b2_stream_ring_result;                    /* 96 bytes */
int  b2_stream_ring_write_enable(b2_ctx* ctx, uint32_t max_bytes, uint32_t max_writes, uint32_t write_out_cap, uint32_t max_segment_size);
int  b2_stream_ring_submit(b2_ctx* ctx, const void* bytes, uint32_t nbytes, const b2_run* runs, uint32_t n_runs,
                           const b2_stream_write_desc* writes, uint32_t n_writes, uint32_t* ticket);
int  b2_stream_ring_wait(b2_ctx* ctx, uint32_t ticket, b2_stream_ring_result* out);

/* ---- counters (bvar::Adder-like, SURVEY §8e): per-GPU totals accumulated by
 * the kernels: [0] in_bytes [1] in_msgs [2] out_bytes [3] out_msgs [4] errors
 * [5] batches [6..7] reserved.  The cross-GPU reduce is an NCCL all-reduce on
 * this int64[8] done by the caller's communicator. -------------------------- */
#define B2_N_COUNTERS 8
int  b2_counters_read(b2_ctx* ctx, int64_t out[B2_N_COUNTERS]);
/* device pointer of the int64[8] (for ncclAllReduce / torch.distributed) */
void* b2_counters_device_ptr(b2_ctx* ctx);
/* bvar's cross-shard sum (an Adder combined over agents, src/bvar/reducer.h:227-233,335) across GPUs: ncclAllReduce(sum, int64 x 8) of the
 * counters IN PLACE on `nccl_comm` (an ncclComm_t of the caller: one rank per GPU) and the ctx's stream; the call returns when the sum is
 * there.  The library does not link NCCL: the entry point is looked up in the running process (torch / the transport loaded it), and the
 * call fails with B2_E_INVAL when it is not there.  Every rank of the communicator must call it. */
int  b2_counters_allreduce(b2_ctx* ctx, void* nccl_comm);

#ifdef __cplusplus
}
#endif
#endif  /* B2RPC_H_ */
