/*
 * simdjson_b200.h -- C ABI of the H100-native simdjson parse engine.
 *
 * This is the drop-in boundary for the ONE hot path of minio/simdjson-go that this
 * library replaces (SURVEY.md section 8b).  The reference has no FFI of its own
 * (pure Go + Go assembly); the seam is
 *
 *     (*internalParsedJson).parseMessage(msg []byte, ndjson bool) error
 *                                                     parse_json_amd64.go:52
 *
 * Everything above it (Parse / ParseND / ParseNDStream, simdjson_amd64.go:66,82,116)
 * and everything that reads its result (Iter / Object / Array / Serializer) stays host
 * code and only sees the output triple { Message, Tape []uint64, Strings.B []byte },
 * which is bit-exact with the reference.  INTEGRATION.md shows the cgo binding.
 *
 * Plain pointers and sizes only: no CUDA or torch types appear in any signature.
 * All functions are thread-safe on distinct contexts; one context serialises its calls.
 */
#ifndef SIMDJSON_B200_H
#define SIMDJSON_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* flags (parse_json_amd64.go:58-62 ndjson; options.go:13 WithCopyStrings) */
#define SJ_FLAG_NDJSON 1u
#define SJ_FLAG_COPY_STRINGS 2u

/* return codes.  Only nil / non-nil matters to the reference's callers; the two parse
 * errors keep the reference's precedence (stage 1 wins, parse_json_amd64.go:123-126). */
#define SJ_OK 0
#define SJ_ERR_STAGE1 1     /* "Failed to find all structural indices for stage 1"  parse_json_amd64.go:93,104 */
#define SJ_ERR_STAGE2 2     /* "Bad parsing while executing stage 2"                parse_json_amd64.go:81,112 */
#define SJ_ERR_NO_DEVICE 3  /* "Host CPU does not meet target specs" analogue       simdjson_amd64.go:43 */
#define SJ_ERR_CAPACITY 4   /* caller buffer too small; *_len hold the required sizes */
#define SJ_ERR_TOO_LARGE 5  /* message longer than SJ_MAX_MESSAGE bytes per call */
#define SJ_ERR_ARGUMENT 6
#define SJ_STREAM_END 7   /* sj_stream_next: input closed and every result delivered (io.EOF, simdjson_amd64.go:189) */
#define SJ_STREAM_EMPTY 8 /* sj_stream_next: nothing handed to a worker yet -- write more (or close the input) */
#define SJ_STREAM_BUSY 9  /* sj_stream_close_input: every slot is in use -- take a result first, then call again */
#define SJ_ERR_EXCHANGE 10 /* sj_parse_nd_sharded_count: a peer's totals did not arrive within the exchange's time limit */
#define SJ_ERR_PEER 11     /* sj_parse_nd_sharded_count: a peer's shard failed before its totals existed (the whole ParseND fails) */
#define SJ_ERR_UNSUPPORTED 12 /* sj_deserialize_device: the stream has S2 or zstd blocks (read them on the CPU) */
/* negative values: -(1000 + cudaError_t) */

#define SJ_MAX_MESSAGE 0x7fffff00ull /* positions are uint32, string lengths keep one flag bit */

typedef struct sj_ctx sj_ctx;

/* simdjson_amd64.go:37 SupportedCPU(): 1 when an sm_90 device is usable */
int sj_supported(void);
int sj_device_count(void);
const char* sj_error_string(int rc);

/* One context = one CUDA stream + reusable device scratch (the analogue of the reused
 * *ParsedJson internals, simdjson_amd64.go:46-51).  device < 0 selects the current device. */
int sj_ctx_create(int device, sj_ctx** out);
void sj_ctx_destroy(sj_ctx* ctx);

/* Stage-2 implementation used by this context: 0 (default) = the streaming kernels (one warp per 6 KiB slab of the
 * message, stage2_stream.cuh) whenever copy_strings is on, 1 = the per-structural kernels (stage2.cuh) always -- the
 * older implementation, kept as the copy_strings = false path and as a second implementation the tests compare with. */
int sj_ctx_set_stage2_impl(sj_ctx* ctx, int impl);

/* Host side of a rank: bind the calling thread (and its future children) to the CPUs of the NUMA node `device` hangs
 * off and prefer that node for memory, so that pinned buffers allocated afterwards sit next to the GPU.  Returns the
 * node, or -1 when the topology is not exposed / nothing was changed. */
int sj_bind_to_device_numa(int device);

/* pinned host memory for callers that want full PCIe speed (optional) */
void* sj_host_alloc(size_t bytes);
void sj_host_free(void* p);

/* Go bytes.TrimSpace as parseMessage applies it (parse_json_amd64.go:55): [*start, *stop) is
 * the trimmed window.  Pure host helper (no device needed). */
void sj_trim_space(const uint8_t* msg, size_t len, size_t* start, size_t* stop);

/* Safe output sizes for a message of `len` bytes (SURVEY.md 8b "ownership"). */
void sj_bounds(size_t len, size_t* tape_cap, size_t* strings_cap);

/*
 * parseMessage replacement (parse_json_amd64.go:52-127), HOST buffers.
 *   msg/len      raw message; trimmed like bytes.TrimSpace; *msg_off / *msg_len give the
 *                trimmed window = ParsedJson.Message (string offsets are relative to it)
 *   tape         receives ParsedJson.Tape   (tape_cap entries available)
 *   strings      receives ParsedJson.Strings.B (strings_cap bytes available)
 * Returns SJ_OK, SJ_ERR_STAGE1, SJ_ERR_STAGE2, SJ_ERR_CAPACITY, ... (see above).
 */
int sj_parse(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, uint64_t* tape, size_t tape_cap,
             size_t* tape_len, uint8_t* strings, size_t strings_cap, size_t* strings_len, size_t* msg_off,
             size_t* msg_len);

/*
 * Same parse with everything resident in device memory (inputs already in HBM, outputs
 * left in HBM): the building block for batch pipelines and what bench.py's `value` times.
 *   d_msg        device pointer, 16-byte aligned, readable up to round_up(len,16); NOT
 *                trimmed by this call (callers pass the trimmed window)
 *   d_tape / d_strings   device output buffers
 */
int sj_parse_device(sj_ctx* ctx, const uint8_t* d_msg, size_t len, uint32_t flags, uint64_t* d_tape, size_t tape_cap,
                    size_t* tape_len, uint8_t* d_strings, size_t strings_cap, size_t* strings_len);

/*
 * ParseND sharded over several GPUs (one process per GPU; SURVEY.md section 8(e)).  ParseND returns ONE ParsedJson
 * whose roots are chained through the whole tape (simdjson_amd64.go:82-93, stage2_build_tape_amd64.go:190-221).
 * Every rank parses a shard of the stream that was cut at record boundaries (every raw '\n' of a valid stream is one:
 * find_quote_mask_and_bits_amd64.s:69-80 rejects control characters inside strings) and passes it TRIMMED, device
 * resident, like sj_parse_device.
 *   1. sj_parse_nd_sharded_count: stage 1 + the counting half of stage 2 on the shard; *totals = its contribution.
 *   2. the ranks exchange the totals (one all-gather of four integers per rank -- NCCL in the caller) and take the
 *      exclusive prefix: msg_base (offset of the shard's trimmed window inside the whole trimmed message; only no-copy
 *      strings use it), tape_base, strings_base.
 *   3. sj_parse_nd_sharded_emit: the emitting half writes the shard's slice of the whole tape / Strings.B into
 *      d_tape[0 .. tape_words) / d_strings[0 .. string_bytes) with every root / scope pointer and string offset
 *      already shifted by the bases: the slices of all ranks, laid end to end, ARE the reference's ParsedJson
 *      (there is no separate rebasing pass over the tape).
 * With one rank and all bases 0 the pair is sj_parse_device.
 */
typedef struct {
    uint64_t msg_bytes;     /* length of the shard as passed in */
    uint64_t tape_words;
    uint64_t string_bytes;
    uint64_t records;       /* roots in the shard */
} sj_shard_totals;
/* d_totals (optional): device memory for the same four integers, written on the context's stream.
 * d_bases (optional): device memory holding { msg_base, tape_base, strings_base }, read by the emitting kernels instead of
 * the three scalar arguments.  With both, and the context running on the caller's stream (sj_ctx_set_stream), the
 * exchange (all-gather + prefix) is enqueued on that stream between the two calls and costs no host round trip. */
int sj_parse_nd_sharded_count(sj_ctx* ctx, const uint8_t* d_msg, size_t len, uint32_t flags, sj_shard_totals* totals,
                              uint64_t* d_totals);
int sj_parse_nd_sharded_emit(sj_ctx* ctx, uint64_t msg_base, uint64_t tape_base, uint64_t strings_base, const uint64_t* d_bases,
                             uint64_t* d_tape, size_t tape_cap, uint8_t* d_strings, size_t strings_cap);
/*
 * The exchange of step 2 as a kernel over peer memory (exchange.cuh) instead of a collective in the caller: the counting
 * half then ENDS with a one-warp kernel that stores this shard's totals into every peer's exchange buffer over NVLink,
 * waits (polling local memory) for the peers' totals and leaves the bases in device memory -- all in front of the
 * counting half's own synchronisation, so the emitting half can be enqueued at once with d_bases = sj_exchange_bases().
 *   sj_exchange_create        allocates this rank's buffer; *handle_out (SJ_EXCHANGE_HANDLE_BYTES, optional) is its CUDA IPC
 *                             handle.  gap_bytes = message bytes between this shard's window and the next shard's (1: the
 *                             newline the shards were cut at; sj_exchange_set_gap changes it for the following calls),
 *                             counted into the msg_base of the ranks behind.  world <= 32.
 *   sj_exchange_connect       handles = world x SJ_EXCHANGE_HANDLE_BYTES, rank r's at offset r (all-gathered by the caller,
 *                             once); opens the peers' buffers (cudaIpcOpenMemHandle).
 *   sj_exchange_connect_ptrs  the same with the peers' buffers already mapped (ranks of one process: sj_exchange_local of
 *                             each context; or symmetric memory the caller owns).
 *   sj_exchange_bases         device pointer to { msg_base, tape_base, strings_base, records_base, whole message bytes,
 *                             whole tape words, whole string bytes, whole records, status, epoch }.
 *   sj_exchange_result        the same ten integers on the host, as of the last sj_parse_nd_sharded_count.
 * Once connected, EVERY sj_parse_nd_sharded_count of the context is a collective call: all ranks make it the same number
 * of times.  A rank whose counting half fails still publishes (a failure marker): its peers' calls return SJ_ERR_PEER.  A
 * peer that never calls makes the others return SJ_ERR_EXCHANGE after the time limit (two seconds by default); no kernel waits forever.
 * Verdicts that only the emitting half finds (stage-2 grammar) stay per rank: the caller combines them.
 */
#define SJ_EXCHANGE_HANDLE_BYTES 64
int sj_exchange_create(sj_ctx* ctx, int rank, int world, uint64_t gap_bytes, void* handle_out);
int sj_exchange_set_gap(sj_ctx* ctx, uint64_t gap_bytes);
int sj_exchange_set_timeout_ms(sj_ctx* ctx, uint32_t ms); /* how long a call waits for its peers (default 2000) */
int sj_exchange_connect(sj_ctx* ctx, const void* handles);
int sj_exchange_connect_ptrs(sj_ctx* ctx, void* const* peer_buffers);
void* sj_exchange_local(sj_ctx* ctx);
const uint64_t* sj_exchange_bases(sj_ctx* ctx);
int sj_exchange_result(sj_ctx* ctx, uint64_t* out10);

/* Run this context's work on the caller's CUDA stream (a cudaStream_t passed as void*; NULL: back to the context's own
 * stream).  For callers that order the parse against their own kernels / collectives without host synchronisation. */
int sj_ctx_set_stream(sj_ctx* ctx, void* cuda_stream);

/*
 * Device-side tape consumers (SURVEY.md section 8(f)): the reference's NDJSON workloads walk
 * the tape right after the parse -- countWhere(key, value, pj) ndjson_test.go:421-459 built
 * on Object.FindKey parsed_object.go:97-140, countObjects ndjson_test.go:461-474, benchmarked
 * as parse + count in BenchmarkNdjsonColdCountStarWithWhere parse_json_amd64_test.go:134-157.
 * Here the walk runs on the tape in HBM, so only two integers travel back over PCIe.
 *   *roots    number of root elements (= countObjects)
 *   *matches  roots whose element is an object whose FIRST member named `key` is a string
 *             equal to `value` (= countWhere)
 * sj_count_where_device: tape / strings / message already in device memory (as left by
 * sj_parse_device; d_msg is only read for no-copy strings).  sj_parse_count_where: HOST
 * message in, parse on the device, count on the device; nothing but the counts is copied back.
 */
int sj_count_where_device(sj_ctx* ctx, const uint8_t* d_msg, const uint64_t* d_tape, size_t tape_len,
                          const uint8_t* d_strings, const uint8_t* key, size_t key_len, const uint8_t* value,
                          size_t value_len, uint64_t* roots, uint64_t* matches);
int sj_parse_count_where(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, const uint8_t* key,
                         size_t key_len, const uint8_t* value, size_t value_len, uint64_t* roots, uint64_t* matches);

/*
 * MarshalJSON on the device: Iter.MarshalJSON of a fresh pj.Iter() (parsed_json.go:394-556), byte for byte.  Every
 * root's value as compact JSON, roots joined by one '\n' (no trailing newline); strings escaped like escapeBytes, floats
 * like appendFloat (shortest round-trip digits; fixed notation for 1e-6 <= |x| < 1e21 and 0, else d.ddde+-N).
 * sj_marshal_device: message, tape, strings and output in device memory; d_msg is only read for no-copy strings.  The
 * tape is checked (tags, links of opens / closes / roots, string ranges, object keys, finite floats): a malformed one
 * returns SJ_ERR_ARGUMENT and nothing outside the three inputs is read.  *out_len = bytes of the text, exact even on
 * SJ_ERR_CAPACITY, when nothing is written.  A tape of length 0 gives 0 bytes.  Tapes longer than SJ_MAX_MARSHAL_TAPE
 * words (the passes keep int32 depths and parents per word) return SJ_ERR_TOO_LARGE.
 * sj_parse_marshal: HOST message in, parse and marshal on the device, only the text is copied to `out` (host memory);
 * parse errors return the parse codes.
 */
#define SJ_MAX_MARSHAL_TAPE 0x7fffffffull
int sj_marshal_device(sj_ctx* ctx, const uint8_t* d_msg, size_t msg_len, const uint64_t* d_tape, size_t tape_len,
                      const uint8_t* d_strings, size_t strings_len, uint8_t* d_out, size_t cap, size_t* out_len);
int sj_parse_marshal(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, uint8_t* out, size_t cap, size_t* out_len);

/*
 * Serializer on the device: the v3 stream of Serializer.Serialize / Deserialize (parsed_serialize.go:200-695) with every
 * block uncompressed (CompressNone), so the reference's NewSerializer().Deserialize reads what these write.  The one
 * intended difference: strings are deduplicated exactly, keeping the first occurrence (the message block holds each
 * distinct string once, in order of first appearance), where the reference's 16 K-bucket table keyed by a per-process
 * seeded hash keeps some duplicates.  The stream does not depend on copy_strings.
 * sj_serialize_device: message, tape, strings and output in device memory.  A tape the reference's Serialize panics on
 * (an unknown tag, a string range outside its buffer, a string or number head as the last word) returns
 * SJ_ERR_ARGUMENT; links are not checked.  *out_len is exact even on SJ_ERR_CAPACITY, when nothing is written.  An empty
 * tape gives the 14-byte empty stream.  Tapes over SJ_MAX_MARSHAL_TAPE words return SJ_ERR_TOO_LARGE.
 * sj_parse_serialize: HOST message in, parse and serialize on the device, only the stream is copied to `out` (host memory).
 * sj_deserialize_device: stream in device memory to tape, Strings.B and message in device memory.  Accepted exactly when
 * the reference's Deserialize on a zeroed tape returns no error and does not panic, every '{' / '[' names a later word
 * that holds its matching close, and no close is named twice; the output then equals the reference's.  Versions 0-3 are
 * read alike and bytes behind the values block are ignored.  S2 / zstd blocks return SJ_ERR_UNSUPPORTED, any other
 * rejection SJ_ERR_ARGUMENT, over SJ_MAX_MARSHAL_TAPE tape words or tags SJ_ERR_TOO_LARGE.  The three sizes are exact on
 * SJ_ERR_CAPACITY; nothing is written unless the call succeeds.
 * sj_test_set_string_hash_bits: keep only `bits` bits of the dedup hash (0 = all), to force hash collisions in tests.
 */
int sj_serialize_device(sj_ctx* ctx, const uint8_t* d_msg, size_t msg_len, const uint64_t* d_tape, size_t tape_len,
                        const uint8_t* d_strings, size_t strings_len, uint8_t* d_out, size_t cap, size_t* out_len);
int sj_parse_serialize(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, uint8_t* out, size_t cap, size_t* out_len);
int sj_deserialize_device(sj_ctx* ctx, const uint8_t* d_in, size_t in_len, uint64_t* d_tape, size_t tape_cap, size_t* tape_len,
                          uint8_t* d_strings, size_t strings_cap, size_t* strings_len, uint8_t* d_msg, size_t msg_cap,
                          size_t* msg_len);
int sj_test_set_string_hash_bits(sj_ctx* ctx, int bits);

/*
 * ParseNDStream (simdjson_amd64.go:116-215) inside the library: the caller pushes the bytes of an
 * NDJSON stream (any host memory, pageable included: they are staged once into pinned buffers),
 * the library cuts them at record boundaries into chunks of about `chunk_bytes` (:157-174; sized
 * to fill a GPU instead of the reference's 10 MiB), parses up to `inflight` chunks concurrently
 * (:132; each on its own context = CUDA stream, so H2D, kernels and D2H overlap) and hands the
 * results out in input order (:134-152), each an independent {Message, Tape, Strings} triple.
 * The first failing chunk ends the stream with its error (:196).  No call blocks on a full
 * pipeline, so one thread can drive it:
 *     while (input left)  { sj_stream_write(s, p, n, &taken); p += taken; n -= taken;
 *                           if (taken == 0) { sj_stream_next(s, &r); ...use r...; sj_stream_release(s, &r); } }
 *     while (sj_stream_close_input(s) == SJ_STREAM_BUSY) { next / release }
 *     while (sj_stream_next(s, &r) == SJ_OK) { ...; sj_stream_release(s, &r); }      // ends with SJ_STREAM_END
 * One writer thread and one reader thread may also run concurrently.
 */
typedef struct sj_stream sj_stream;
typedef struct {
    const uint8_t* message;  /* trimmed chunk = ParsedJson.Message (no-copy string offsets index into it) */
    size_t message_len;
    const uint64_t* tape;    /* ParsedJson.Tape */
    size_t tape_len;
    const uint8_t* strings;  /* ParsedJson.Strings.B */
    size_t strings_len;
    uint64_t seq;            /* chunk number in input order */
    void* slot;              /* owner of the (pinned) buffers above; valid until sj_stream_release */
} sj_stream_result;
int sj_stream_create(int device, int inflight, size_t chunk_bytes, uint32_t flags, sj_stream** out);
void sj_stream_destroy(sj_stream* s);
int sj_stream_write(sj_stream* s, const uint8_t* data, size_t len, size_t* taken);
int sj_stream_close_input(sj_stream* s);
int sj_stream_next(sj_stream* s, sj_stream_result* res);
int sj_stream_release(sj_stream* s, const sj_stream_result* res);

/*
 * K0: the synthetic NDJSON stream of the benchmark (SURVEY.md 8d, S3), generated on the device: record g is line
 * (g mod L) of `tmpl` (L records separated by '\n', each starting with {"Ticket":"<10 digits>" -- the reference's
 * parking-citations fixture) with the ten digits replaced by g, zero padded.  Writes records first_record ..
 * first_record + n_records - 1 joined by '\n' into d_out (device memory, 16-byte aligned); first_record must be a
 * multiple of L.  *out_len = bytes written (exact even on SJ_ERR_CAPACITY).
 */
int sj_gen_ndjson_device(sj_ctx* ctx, const uint8_t* tmpl, size_t tmpl_len, uint64_t first_record, uint64_t n_records,
                         uint8_t* d_out, size_t cap, size_t* out_len);

/*
 * Stage 1 + flatten only (findStructuralIndices, stage1_find_marks_amd64.go:41):
 * writes the concatenated uint32 index deltas the reference would hand to stage 2
 * (flatten_bits_amd64.s:26-60: delta to the previous structural, first = position+1).
 * HOST buffers; msg is used as given (no trimming).  *n is exact even on SJ_ERR_CAPACITY.
 * Returns SJ_OK or SJ_ERR_STAGE1 (indices are still written), ...
 */
int sj_find_structural_indices(sj_ctx* ctx, const uint8_t* msg, size_t len, int ndjson, uint32_t* deltas,
                               size_t cap, size_t* n);

/* Device-resident stage 1: positions (deltas = 0) or deltas (deltas = 1) into d_out. */
typedef struct {
    uint64_t n_idx;
    uint32_t error;          /* control character inside a string */
    uint32_t ends_in_string;
    uint32_t last_pos;
    uint32_t overflow;
} sj_stage1_info;
int sj_stage1_device(sj_ctx* ctx, const uint8_t* d_msg, size_t len, int ndjson, int deltas, uint32_t* d_out,
                     size_t cap, sj_stage1_info* info);
/* asynchronous launch of the same kernel on the context's stream (no result read-back);
 * used by bench.py to time the kernel alone with CUDA events */
int sj_stage1_launch(sj_ctx* ctx, const uint8_t* d_msg, size_t len, int ndjson, int deltas, uint32_t* d_out,
                     size_t cap);
/* CUDA-event timing helpers on the context's stream (bench only) */
int sj_ctx_sync(sj_ctx* ctx);
int sj_event_record(sj_ctx* ctx, int which /*0 = start, 1 = stop*/);
int sj_event_elapsed_ms(sj_ctx* ctx, float* ms);
int sj_kernel_launches(sj_ctx* ctx, uint64_t* count); /* kernels launched by this context so far */

/* ---- unit-test hooks: the reference's per-routine Go stubs replayed on the device code ----
 * find_subroutines_amd64.go:26-231.  For block i: in = blocks + 64*i and
 * carry_in[4*i..] = { prev_iter_ends_odd_backslash, prev_iter_inside_quote (0 / ~0),
 * prev_iter_ends_pseudo_pred, ndjson }.  out[12*i..] = { odd_ends, quote_mask, quote_bits,
 * error_mask, whitespace, structurals(raw), structurals_finalized (incl. newlines if
 * ndjson), raw newline mask (before & ~quote_mask), carry_out odd_backslash, carry_out inside_quote, carry_out
 * pseudo_pred, any-control-character flag }.  Host buffers. */
int sj_test_block_masks(sj_ctx* ctx, const uint8_t* blocks, size_t nblocks, const uint64_t* carry_in, uint64_t* out);
/* geometry of the stage-1 kernel, for tests that aim carries at its edges: out = { block bytes (64), step bytes (one
 * warp pass: 32 blocks), slab bytes (one warp's share of a tile), tile bytes (one CTA iteration = one look-back) } */
void sj_test_geometry(uint32_t out[4]);
/* finalize_structurals on caller-provided masks: in[5*i..] = {structurals, whitespace,
 * quote_mask, quote_bits, prev_pseudo}; out[2*i..] = {structurals, prev_pseudo'} */
int sj_test_finalize(sj_ctx* ctx, const uint64_t* in, size_t n, uint64_t* out);
/* flatten_bits_incremental over a sequence of 64-bit masks (flatten_bits_amd64.s:26),
 * carried = 0 and position = ^0 initially */
int sj_test_flatten_bits(sj_ctx* ctx, const uint64_t* masks, size_t nmasks, uint32_t* deltas, size_t cap, size_t* n);
/* parse_string_validate_only + parse_string (parse_string_amd64.go:33,48) for a batch:
 * string i = buf[offs[i] .. offs[i+1]) starting AT its opening quote; max_size[i] is
 * maxStringSize.  ok[i], src_len[i], dst_len[i]; unescaped bytes are written at
 * dst + offs[i].  Host buffers. */
int sj_test_parse_strings(sj_ctx* ctx, const uint8_t* buf, const uint64_t* offs, size_t n, const uint64_t* max_size,
                          uint8_t* ok, uint64_t* src_len, uint64_t* dst_len, uint8_t* dst);
/* parseNumber (parse_number.go:65) for a batch: number i = buf[offs[i] .. offs[i+1]);
 * tag[i] = tape tag word (tag << 56 | flags, 0 on failure), val[i] = raw value */
int sj_test_parse_numbers(sj_ctx* ctx, const uint8_t* buf, const uint64_t* offs, size_t n, uint64_t* tag,
                          uint64_t* val);

#ifdef __cplusplus
}
#endif
#endif
