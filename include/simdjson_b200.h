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
#define SJ_ERR_UNSUPPORTED 12 /* sj_deserialize_device: S2 blocks in SJ_COMPRESS_NONE mode, zstd blocks in SJ_COMPRESS_NONE /
                                 SJ_COMPRESS_FAST mode (set SJ_COMPRESS_DEFAULT or SJ_COMPRESS_BEST to read them) */
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
 * ForEach + FindElement on the device: for every root of a tape (in tape order: one per NDJSON record, one for a single
 * document) and every path, the value at that path, read into typed columns in device memory.  A cell is a literal
 * port of ParsedJson.ForEach (parsed_json.go:125-138) handing each root's element to Iter.FindElement(path...)
 * (:833-864 -> Iter.Object :998-1018 -> Object.FindPath parsed_object.go:256-316), then the accessor of the path's kind:
 *   SJ_FIND_KIND_ELEMENT  none               SJ_FIND_KIND_INT64   Iter.Int    (:629-661)
 *   SJ_FIND_KIND_UINT64   Iter.Uint (:679-712) SJ_FIND_KIND_FLOAT64 Iter.Float (:560-583)
 *   SJ_FIND_KIND_BOOL     Iter.Bool (:867-875) SJ_FIND_KIND_STRING  Iter.StringBytes (:741-749)
 *   SJ_FIND_KIND_JSON     Element.Iter.MarshalJSON (:394-556): the element as compact JSON text, byte for byte what the
 *                         reference writes (strings escaped like escapeBytes, floats like appendFloat); a scalar gives
 *                         its own text ("abc", 12, true).  Its number is 7: 6 stays an unknown kind (SJ_ERR_ARGUMENT).
 *   SJ_FIND_KIND_STRING_CVT  Iter.StringCvt (:775-799): strings raw (not escaped), int64 / uint64 in decimal, true /
 *                         false / null as written, floats as appendFloat (an INF or NaN is SJ_FIND_CONVERT)
 *   list kinds (sj_find_lists_device / sj_parse_find_lists only): Iter.Array (:1022-1039), then
 *   SJ_FIND_KIND_ARRAY_FLOAT64  Array.AsFloat (parsed_array.go:145-181)  SJ_FIND_KIND_ARRAY_INT64  Array.AsInteger (:185-232)
 *   SJ_FIND_KIND_ARRAY_UINT64   Array.AsUint64 (:236-283)     SJ_FIND_KIND_ARRAY_STRING Array.AsString (:287-314)
 *   SJ_FIND_KIND_ARRAY_STRING_CVT  Array.AsStringCvt (:319-344): each element as SJ_FIND_KIND_STRING_CVT
 * So the first member with the key decides, keys compare on their unescaped bytes, arrays are never entered, and a
 * root or intermediate value that is not an object is SJ_FIND_NOT_OBJECT, not SJ_FIND_NOT_FOUND.  Where amd64 Go and
 * CUDA's conversions differ the cell follows Go: Int() of a float of exactly 2^63 is math.MinInt64 (CVTTSD2SQ), Uint()
 * of exactly 2^64 is 1<<63 (Go's float64ToUint64 lowering).
 * Cell status (u8): SJ_FIND_OK found and converted; SJ_FIND_NOT_FOUND ErrPathNotFound (also a path of 0 segments);
 * SJ_FIND_NOT_OBJECT "type ... found before object" / "value of key ... is not an object"; SJ_FIND_CONVERT the accessor's
 * error; SJ_FIND_CORRUPT any other error (or panic) of the reference on a malformed tape.  Tag (u8): the found element's
 * tag byte; index (i64): the tape index of its head word (-1 and tag 0 when nothing was found); value (8 bytes): int64,
 * uint64, the bits of a float64, 0 / 1 for BOOL, the byte length for STRING and JSON, 0 for ELEMENT and for cells not OK.
 * A JSON cell is SJ_FIND_CONVERT when the element is TypeNone (the key's value is missing at the very end of a malformed
 * tape: MarshalJSON's "no content queued in iterator"), and SJ_FIND_CORRUPT when its sub-tree, the words [index, index +
 * its restricted tape length), fails the checks sj_marshal_device applies (tags, open / close links, string ranges,
 * object keys, finite floats), or holds a root ('r') or nop ('N') word.  This is stricter than the reference's walk, as
 * the whole-tape marshal is; the checks read the sub-tree alone, so a malformed region elsewhere on the tape leaves a
 * cell whose own sub-tree is well formed unchanged.
 * Layout, path-major with a row stride of row_cap: cell (p, r) of status / tag / index / value is at p * row_cap + r;
 * STRING and JSON path s (counting those paths only, in path order) has str_offsets[s * (row_cap + 1) + r], r = 0 ..
 * rows, into str_bytes, so row r's bytes are [off[r], off[r + 1]) (with no rows, the one entry 0 is written when
 * str_offsets is given).  A call without JSON paths writes what it wrote before they existed.
 * A list cell is SJ_FIND_OK when the element is an array and the accessor returns no error; its value is the element
 * count (a STRING_CVT cell's is the byte length).  SJ_FIND_CONVERT: a fresh Element, "next item is not array", "unable
 * to convert type", an overflow / underflow / negative value, "element in array is not string", StringCvt's "cannot
 * convert type" and appendFloat's INF / NaN.  SJ_FIND_CORRUPT: "extended beyond tape", "no more values", AdvanceIter's
 * errors, a string range outside its buffer and any index out of range.  The first failing element decides, and a cell
 * that is not OK has no elements and no bytes.  The port is literal: AsFloat / AsInteger / AsUint64 read tag words at
 * even offsets from the word after '[', so a nop or a nested '[' / '{' there is SJ_FIND_CONVERT and a read past the
 * array's tape is SJ_FIND_CORRUPT; AsString / AsStringCvt step with AdvanceIter, so nops are skipped (a skip of 0 is
 * SJ_FIND_CORRUPT), a nested scope is stepped over by its link and then rejected, and the first TypeNone tag (']', or any
 * unknown tag) ends the list as OK.  AsInteger of a float of exactly 2^63 is math.MinInt64; AsUint64 rejects floats
 * above 2^63 (Iter.Uint accepts them up to 2^64) and makes exactly 2^63 (and NaN) 1<<63.  The work is spread over the
 * array words, not over cells; only a cell whose AdvanceIter walk meets a nop word (foreign or Deserialize'd tapes) is
 * finished by one thread, from that word on.
 * List layout (sj_find_lists_out): list path l (counting list paths only, in path order) has offsets[l * (row_cap + 1)
 * + r], r = 0 .. rows, into one pool `elems` shared by all list paths in path then row order, so row r's elements are
 * elems[off[r] .. off[r + 1]): int64 / uint64 / float64 bits, and for ARRAY_STRING / ARRAY_STRING_CVT each element's
 * byte length.  STRING_CVT, ARRAY_STRING and ARRAY_STRING_CVT paths are variable-length byte columns like STRING and
 * JSON paths (numbered with them, in path order); a string list row's bytes are its elements back to back, element k
 * starting at the row's str_offsets entry plus the lengths of elements 0 .. k-1.
 * Limits: 1 to 64 paths, 0 to 32 segments each, 16 KiB of segment bytes in all; else SJ_ERR_ARGUMENT.  A tape longer
 * than 2^32 - 1 words returns SJ_ERR_TOO_LARGE, and so does a JSON or list path whose cells cover more than SJ_MAX_MARSHAL_TAPE
 * tape words in all (only a malformed tape's cells can overlap, so on any other tape this is within the tape).  *rows and *str_bytes are exact even on SJ_ERR_CAPACITY (rows > row_cap
 * or str_bytes > str_cap), when nothing is written; out may be NULL to ask for the sizes.
 * sj_find_device: message, tape, strings and out in device memory, with their lengths (every read stays inside them).
 * On the tape this context's last parse left in HBM the rows are stage 2's root list, until the next parse or an
 * sj_deserialize_device that writes over any part of that tape (after either it is a foreign tape); on any other
 * tape they are found on the device: the 'r' words that point forward and are not the value word of a string or number (read from word 0),
 * which on every tape the parser or sj_deserialize_device writes are the roots ForEach visits.  sj_parse_find: HOST message in, parse and find on the device, only the columns are copied to `out`
 * (host memory); parse errors return the parse codes.
 * sj_find_device / sj_parse_find accept every kind but the list kinds (8-12), which return SJ_ERR_ARGUMENT there.
 * sj_find_lists_device / sj_parse_find_lists take the same arguments plus the list output and *elems (the pool's
 * element total); *rows, *str_bytes and *elems are exact even on SJ_ERR_CAPACITY (elems > elem_cap too), when nothing is
 * written, and `lists` may be NULL to ask for the sizes.  Without list paths they compute what the two above compute.
 */
#define SJ_FIND_OK 0
#define SJ_FIND_NOT_FOUND 1
#define SJ_FIND_NOT_OBJECT 2
#define SJ_FIND_CONVERT 3
#define SJ_FIND_CORRUPT 4
#define SJ_FIND_KIND_ELEMENT 0
#define SJ_FIND_KIND_INT64 1
#define SJ_FIND_KIND_UINT64 2
#define SJ_FIND_KIND_FLOAT64 3
#define SJ_FIND_KIND_BOOL 4
#define SJ_FIND_KIND_STRING 5
#define SJ_FIND_KIND_JSON 7
#define SJ_FIND_KIND_ARRAY_FLOAT64 8
#define SJ_FIND_KIND_ARRAY_INT64 9
#define SJ_FIND_KIND_ARRAY_UINT64 10
#define SJ_FIND_KIND_ARRAY_STRING 11
#define SJ_FIND_KIND_ARRAY_STRING_CVT 12
#define SJ_FIND_KIND_STRING_CVT 13
typedef struct {
    const uint8_t* segments;   /* the key segments laid end to end (host memory) */
    const uint32_t* seg_lens;  /* n_segments lengths */
    uint32_t n_segments;
    uint32_t kind;             /* SJ_FIND_KIND_* */
} sj_find_path;
typedef struct {
    uint8_t* status;       /* [n_paths][row_cap] */
    uint8_t* tag;          /* [n_paths][row_cap] */
    int64_t* index;        /* [n_paths][row_cap] */
    uint64_t* value;       /* [n_paths][row_cap] */
    int64_t* str_offsets;  /* [STRING paths][row_cap + 1] */
    uint8_t* str_bytes;    /* str_cap bytes */
    size_t row_cap;
    size_t str_cap;
} sj_find_out;
int sj_find_device(sj_ctx* ctx, const uint8_t* d_msg, size_t msg_len, const uint64_t* d_tape, size_t tape_len,
                   const uint8_t* d_strings, size_t strings_len, const sj_find_path* paths, size_t n_paths,
                   const sj_find_out* out, size_t* rows, size_t* str_bytes);
int sj_parse_find(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, const sj_find_path* paths, size_t n_paths,
                  const sj_find_out* out, size_t* rows, size_t* str_bytes);
typedef struct {
    int64_t* offsets;  /* [list paths][row_cap + 1]: row r's elements are elems[offsets[r] .. offsets[r + 1]) */
    uint64_t* elems;   /* elem_cap words: int64 / uint64 / float64 bits; for string lists each element's byte length */
    size_t elem_cap;
} sj_find_lists_out;
int sj_find_lists_device(sj_ctx* ctx, const uint8_t* d_msg, size_t msg_len, const uint64_t* d_tape, size_t tape_len,
                         const uint8_t* d_strings, size_t strings_len, const sj_find_path* paths, size_t n_paths,
                         const sj_find_out* out, const sj_find_lists_out* lists, size_t* rows, size_t* str_bytes,
                         size_t* elems);
int sj_parse_find_lists(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, const sj_find_path* paths, size_t n_paths,
                        const sj_find_out* out, const sj_find_lists_out* lists, size_t* rows, size_t* str_bytes, size_t* elems);

/*
 * Array rows of the find: Array.ForEach over every record's array at a row path, each element one row of the find's
 * columns.  A record is a root, in the find's order.  Its array is a literal port of ParsedJson.ForEach's element
 * (parsed_json.go:125-138) handed to FindElement(row_path...) (:833-864) and Element.Iter.Array (:1022-1039); a row
 * path of 0 segments takes elem.Array directly (root arrays, NDJSON lines that are arrays), the one place where 0
 * segments is not ErrPathNotFound.  The row path's kind must be SJ_FIND_KIND_ELEMENT; it has the limits of a path.
 * Record status (u8, the list cells' codes): SJ_FIND_OK an array; SJ_FIND_NOT_FOUND FindElement found nothing;
 * SJ_FIND_NOT_OBJECT it met a value that is not an object; SJ_FIND_CONVERT "next item is not array" or a fresh Element;
 * SJ_FIND_CORRUPT a malformed tape.  A record that is not OK has no rows.
 * Rows: the elements Array.ForEach (parsed_array.go:45-56) hands its callback, in order: Advance (:196-223) from the
 * word after '[' over the array's tape Tape[:end], until TypeNone, quirks included: a nop skips 1 + its skip words (one
 * more than AdvanceInto), a scope whose link lies behind it, ']', '}', any unknown tag and the end of the array's tape
 * end the walk silently (ForEach has no error: the walk never makes a record CORRUPT), and an 'r' is an element.
 * Cells: each (path, row) cell is the find's cell computed from the element's Iter instead of a root: FindElement(path...)
 * enters a '{' through Iter.Object with the array's tape as its tape, an 'r' through Root, anything else is
 * SJ_FIND_NOT_OBJECT and a path of 0 segments SJ_FIND_NOT_FOUND; then the accessor of every kind, list kinds included.
 * Status, tag, index, value, the byte columns and the list pool follow the find's contract above with rows = elements
 * (row_cap = out->row_cap); `lists` may be NULL when no path has a list kind.
 * Layout (sj_find_rows_out): record k's rows are [rec_offsets[k], rec_offsets[k + 1]) (rec_offsets[0] = 0, also with no
 * records), row_tag / row_index the tag byte and tape index of each row's element head.  *records, *rows, *str_bytes and
 * *elems are exact even on SJ_ERR_CAPACITY (records > record_cap, rows > row_cap, str_bytes > str_cap or elems >
 * elem_cap), when nothing is written; out, lists and rows_out may be NULL to ask for the sizes.  The array words of all
 * records above SJ_MAX_MARSHAL_TAPE return SJ_ERR_TOO_LARGE, as for list paths.
 * The enumeration runs over the array words, not over records: the heads directly inside each array are proposed as its
 * elements, and each checks that Advance's successor of the one in front of it is itself; a record that fails a check or
 * meets a nop is walked by one thread.  Launches: KR1 and 4 for the records' word scan, 8 over the array words (none
 * without them), KR5 and 4 for the row counts' scan, KR6, KR7 and KR8 (21 with array words), with two read-backs, then
 * the find's passes over the rows (5 with scalar paths); a foreign tape adds the find's 7 that find its roots.
 * sj_find_rows_device: as sj_find_device (device memory).  sj_parse_find_rows: as sj_parse_find (HOST message, parse
 * codes on a parse error, only the columns are copied back, into host memory).
 */
typedef struct {
    uint8_t* rec_status;   /* [record_cap]: the row path's cell per record */
    int64_t* rec_offsets;  /* [record_cap + 1]: record k's rows are [rec_offsets[k], rec_offsets[k + 1]) */
    uint8_t* row_tag;      /* [row_cap]: the tag byte of each row's element */
    int64_t* row_index;    /* [row_cap]: the tape index of each row's element head */
    size_t record_cap;
} sj_find_rows_out;
int sj_find_rows_device(sj_ctx* ctx, const uint8_t* d_msg, size_t msg_len, const uint64_t* d_tape, size_t tape_len,
                        const uint8_t* d_strings, size_t strings_len, const sj_find_path* row_path, const sj_find_path* paths,
                        size_t n_paths, const sj_find_out* out, const sj_find_lists_out* lists, const sj_find_rows_out* rows_out,
                        size_t* records, size_t* rows, size_t* str_bytes, size_t* elems);
int sj_parse_find_rows(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, const sj_find_path* row_path,
                       const sj_find_path* paths, size_t n_paths, const sj_find_out* out, const sj_find_lists_out* lists,
                       const sj_find_rows_out* rows_out, size_t* records, size_t* rows, size_t* str_bytes, size_t* elems);
/* test hook: how many records of this context's last array-rows or member-rows call failed the propose / verify checks
 * and were walked by one thread (0 on every tape the parser writes) */
int sj_test_find_rows_serial(sj_ctx* ctx, uint64_t* records);

/*
 * Member rows of the find: Object.ForEach over every record's object at a row path, each member one row of the find's
 * columns, with its key in a column of its own.  Records as for the array rows, with Element.Iter.Object
 * (parsed_json.go:998-1018) in place of Iter.Array: SJ_FIND_CONVERT "next item is not object" or a fresh Element;
 * SJ_FIND_CORRUPT "object ends at index before start" or "object extended beyond tape".  A row path of 0 segments takes
 * elem.Object directly (root objects, NDJSON records: every key of every record).
 * Rows: the members for which Object.ForEach(fn, onlyKeys) (parsed_object.go:142-186) calls fn, in order, over the
 * object's tape Tape[:end] with Advance: a key position or a value of TypeNone ('}', ']', an unknown tag, a scope whose
 * link lies behind it, the end of the tape) ends the walk silently, a nop is skipped as Advance skips it, a key that is
 * not a string or has no two words behind it inside the tape ("unexpected name tag") or whose bytes lie outside their
 * buffer ("getting object name") makes the record SJ_FIND_CORRUPT.  The rows fn received in front of that error stay:
 * this is the one case where a record that is not OK has rows.  only_keys (kind SJ_FIND_KIND_ELEMENT, a path's limits:
 * at most 32 keys, 16 KiB; NULL or 0 segments: every key) is onlyKeys: a member whose key is not among its segments is
 * skipped, and the walk ends at the match whose count equals the number of distinct segments (matches are counted, so a
 * key that occurs twice is two rows).
 * Cells: a path of >= 1 segment is the array rows' cell from the Iter fn receives; a path of 0 segments is the member's
 * value itself, the element Object.FindPath returns when it stops at this member (AdvanceIter from the key,
 * parsed_object.go:298-303), with every kind applied to it.  rows_out is the array rows' layout with row_tag / row_index
 * of each member's value head.
 * Keys (sj_find_keys_out): row r's key is key_bytes[key_offsets[r], key_offsets[r + 1]), unescaped as stringByteAt
 * returns it (from Strings.B, or from the message for no-copy strings); key_offsets has row_cap + 1 entries (key_offsets[0]
 * = 0, also with no rows).  *records, *rows, *str_bytes, *elems and *key_bytes are exact even on SJ_ERR_CAPACITY (also
 * key_bytes > key_cap), when nothing is written; every output may be NULL to ask for the sizes.  The object words of all
 * records above SJ_MAX_MARSHAL_TAPE return SJ_ERR_TOO_LARGE.
 * The enumeration is the array rows' over the object words; each candidate's rank in its record tells key from value,
 * and the selected keys are counted by a scan of their own.  Launches: the array rows' with 3 more over the object words
 * (KO1 and its scan), KO2 in place of KR6, and for rows > 0 4 for the key lengths' scan with a read-back and KO3.
 * sj_find_members_device: as sj_find_rows_device (device memory).  sj_parse_find_members: as sj_parse_find_rows.
 */
typedef struct {
    int64_t* key_offsets;  /* [row_cap + 1]: row r's key is key_bytes[key_offsets[r] .. key_offsets[r + 1]) */
    uint8_t* key_bytes;    /* key_cap bytes */
    size_t key_cap;
} sj_find_keys_out;
int sj_find_members_device(sj_ctx* ctx, const uint8_t* d_msg, size_t msg_len, const uint64_t* d_tape, size_t tape_len,
                           const uint8_t* d_strings, size_t strings_len, const sj_find_path* row_path,
                           const sj_find_path* only_keys, const sj_find_path* paths, size_t n_paths, const sj_find_out* out,
                           const sj_find_lists_out* lists, const sj_find_rows_out* rows_out, const sj_find_keys_out* keys_out,
                           size_t* records, size_t* rows, size_t* str_bytes, size_t* elems, size_t* key_bytes);
int sj_parse_find_members(sj_ctx* ctx, const uint8_t* msg, size_t len, uint32_t flags, const sj_find_path* row_path,
                          const sj_find_path* only_keys, const sj_find_path* paths, size_t n_paths, const sj_find_out* out,
                          const sj_find_lists_out* lists, const sj_find_rows_out* rows_out, const sj_find_keys_out* keys_out,
                          size_t* records, size_t* rows, size_t* str_bytes, size_t* elems, size_t* key_bytes);

/*
 * MarshalJSON on the device: Iter.MarshalJSON of a fresh pj.Iter() (parsed_json.go:394-556), byte for byte.  Every
 * root's value as compact JSON, roots joined by one '\n' (no trailing newline); strings escaped like escapeBytes, floats
 * like appendFloat (shortest round-trip digits; fixed notation for 1e-6 <= |x| < 1e21 and 0, else d.ddde+-N).
 * sj_marshal_device: message, tape, strings and output in device memory; d_msg is only read for no-copy strings.  The
 * tape is checked (tags, links of opens / closes / roots, string ranges, object keys, finite floats): a malformed one
 * returns SJ_ERR_ARGUMENT and nothing outside the three inputs is read.  *out_len = bytes of the text, exact even on
 * SJ_ERR_CAPACITY, when nothing is written.  A tape of length 0 gives 0 bytes.  Tapes longer than SJ_MAX_MARSHAL_TAPE
 * words (the passes keep int32 depths and parents per word) return SJ_ERR_TOO_LARGE.  The same bound holds for the
 * words one SJ_FIND_KIND_JSON path's cells cover in sj_find_device / sj_parse_find.
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
 * read alike and bytes behind the values block are ignored.  S2 / zstd blocks return SJ_ERR_UNSUPPORTED (they are
 * read in the compressed modes, below), any other
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
 * Serializer.CompressMode (parsed_serialize.go:93-115) of a context's Serializer calls.  SJ_COMPRESS_NONE (the default):
 * the streams and the Deserialize verdicts above.  SJ_COMPRESS_FAST: sj_serialize_device / sj_parse_serialize write the
 * message, tags and values blocks as block type 1, an S2 stream each (s2.cuh), and sj_deserialize_device reads S2 blocks
 * too; zstd blocks stay SJ_ERR_UNSUPPORTED in SJ_COMPRESS_NONE and SJ_COMPRESS_FAST mode.  SJ_COMPRESS_DEFAULT: the
 * tags block is written as block type 2, a zstd frame (zstd.cuh), the message and values blocks as S2; SJ_COMPRESS_BEST:
 * all three as zstd.  Both read uncompressed, S2 and zstd blocks.  Any other mode is SJ_ERR_ARGUMENT.
 * An S2 block written here: the stream identifier ff 06 00 00 "S2sTwO" (no bytes at all for an empty block), then one
 * chunk per 64 KiB of input, compressed (0x00, literals and copies with 1- and 2-byte offsets only: the Snappy subset)
 * or stored (0x01) when compressing would not make it shorter, each with the masked CRC-32C of its bytes.  The stream
 * is deterministic: it depends only on the tape's content, as the uncompressed one does.
 * An S2 block read here, after the header checks above, is accepted as s2.Reader fills the block's uncompressed size:
 * the first chunk is an identifier ("S2sTwO", or "sNaPpY": then no chunk may decode to more than 64 KiB), which may
 * repeat; 0x00 / 0x01 chunks are at least 4 bytes long, decode to at most 4 MiB, in full, to their stated length and CRC;
 * 0x80 - 0xfe chunks are skipped, 0x02 - 0x7f rejected; blocks are S2 (copy offset 0 of a 1-byte-offset copy repeats
 * the last offset).  Chunks are read until the size is filled and nothing behind that chunk is read; running out of
 * chunks first is rejected; a block of size 0 reads nothing.  Every such rejection is SJ_ERR_ARGUMENT.  A stream is
 * accepted exactly when it is accepted with each S2 block replaced by its inflated bytes as an uncompressed block.
 * sj_test_s2_encode / sj_test_s2_decode: the codec alone on device buffers -- one S2 stream of `in` (identifier and
 * chunks; *out_len exact on SJ_ERR_CAPACITY), and one S2 stream read as a block of `want` uncompressed bytes.
 * A zstd block written here: nothing for an empty block (as the S2 path writes nothing: both read back as empty), else
 * one frame -- single segment, Frame_Content_Size present, no checksum, no dictionary -- of one block per 64 KiB of
 * input, the last flagged: a compressed block (raw literals, sequences with the predefined LL / OF / ML tables and new
 * offsets only, matches inside the block) or a raw block when compressing would not make it shorter.  Deterministic.
 * A zstd block read here (RFC 8878; the reference's decoder.DecodeAll and then the size check) is accepted when:
 *  - frames: zero or more back to back fill the block exactly, each a zstd frame (magic 28 b5 2f fd) or a skippable
 *    frame (magic 0x184D2A50 - 0x184D2A5F, skipped); all frames together decode to the block's uncompressed size;
 *  - frame header: reserved bit 0; dictionary ID absent or 0; Frame_Content_Size, when present, equals the frame's
 *    output; the window is the descriptor's, or the content size of a single-segment frame; with the checksum flag,
 *    the low 32 bits of XXH64 (seed 0) of the frame's output match;
 *  - blocks: raw, RLE and compressed (reserved type 3 rejected); a compressed block's content and decoded size at
 *    most min(window, 128 KiB); raw and RLE blocks are not limited (see below); the last-block flag ends the frame;
 *  - literals: raw, RLE, Huffman and treeless (the last Huffman table of the same frame, none: rejected), one stream or
 *    four with the jump table; weights FSE-compressed or in the direct 4-bit form, at most 11 bits, completing a tree;
 *  - sequences: every count encoding; predefined, RLE, FSE and repeat modes (repeat: a table of an earlier block of
 *    the same frame); FSE descriptions whose counts add up exactly; literal lengths within the literals; every
 *    bitstream (Huffman streams, FSE weights aside, and the sequences) ending exactly at its padding; a block with no
 *    sequences ends behind its count byte;
 *  - offsets: repeat offsets start at 1, 4, 8 in each frame; with literal length 0 a repeat code shifts by one (1 is
 *    rep2, 2 rep3, 3 rep1 - 1, rejected when that is 0, as libzstd rejects it); a match reaching in front of the frame's
 *    first byte is rejected (no dictionary).
 * These rules are RFC 8878's and were checked against libzstd (through pyarrow) only; where the reference's Go decoder
 * may differ from it -- the windows it refuses, an offset beyond the window inside the frame, a literal count below 6
 * with four streams, FSE weights over 255 symbols -- this follows the RFC.  Two rules follow libzstd instead of the
 * RFC: raw and RLE blocks larger than min(window, 128 KiB) are accepted (RFC 8878 3.1.1.2.2 limits every block type;
 * libzstd limits compressed blocks only), and rep1 - 1 = 0 is rejected.  Every rejection is SJ_ERR_ARGUMENT; a stream
 * whose zstd blocks end more than 4 GiB into the inflated stream returns SJ_ERR_TOO_LARGE (the decoder's per-byte
 * sources are 32-bit positions).  A stream is accepted exactly when
 * it is accepted with each compressed block replaced by its inflated bytes as an uncompressed block.
 * sj_test_zstd_encode / sj_test_zstd_decode: the zstd codec alone, shaped like the S2 hooks: one frame of `in`, and
 * zstd frames read as a block of `want` uncompressed bytes.
 */
#define SJ_COMPRESS_NONE 0
#define SJ_COMPRESS_FAST 1
#define SJ_COMPRESS_DEFAULT 2
#define SJ_COMPRESS_BEST 3
int sj_ctx_set_compress_mode(sj_ctx* ctx, int mode);
int sj_test_s2_encode(sj_ctx* ctx, const uint8_t* d_in, size_t len, uint8_t* d_out, size_t cap, size_t* out_len);
int sj_test_s2_decode(sj_ctx* ctx, const uint8_t* d_in, size_t len, uint8_t* d_out, size_t want, size_t* got);
int sj_test_zstd_encode(sj_ctx* ctx, const uint8_t* d_in, size_t len, uint8_t* d_out, size_t cap, size_t* out_len);
int sj_test_zstd_decode(sj_ctx* ctx, const uint8_t* d_in, size_t len, uint8_t* d_out, size_t want, size_t* got);
/*
 * sj_test_stage2_internal: the internal-error word of the last parse through the streaming stage 2 (copy_strings):
 * non-zero when the tape writer's counts of a slab differed from the ones stage 1 added up for it (the parse then
 * returns SJ_ERR_STAGE2).  A defect of the library, never a verdict on the input: tests expect 0 on every input.
 */
int sj_test_stage2_internal(sj_ctx* ctx, uint32_t* word);
/*
 * sj_test_stage1_ctas: the CTAs of stage 1's cooperative grid on the context's device (one per SM).  Stage 1 deals its
 * tiles round-robin over them, so tests place documents on the edge of a grid round with it.
 */
int sj_test_stage1_ctas(sj_ctx* ctx, uint32_t* ctas);

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
