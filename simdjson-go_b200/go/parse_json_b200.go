//go:build cgo && b200

// Package simdjson: drop-in replacement for parse_json_amd64.go of minio/simdjson-go.
//
// This file is the ONLY Go code the GPU path needs: it replaces
// (*internalParsedJson).parseMessage (reference parse_json_amd64.go:52) with one cgo call into
// libsimdjson_b200.so.  Parse / ParseND / ParseNDStream (simdjson_amd64.go:66,82,116) and every
// tape consumer (Iter, Object, Array, Serializer) stay as they are: the {Message, Tape,
// Strings.B} triple written here is bit-exact with the assembly path.
//
// NOTE: the build image of this repository has no Go toolchain, so this file is not compiled
// by the test-suite; the identical call sequence is exercised through the ctypes binding
// (simdjson-go_b200/simdjson_b200/__init__.py: Context.parse).  Build it inside a checkout of
// the reference with:  go build -tags b200   (and drop parse_json_amd64.go's build tag).
package simdjson

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/.. -lsimdjson_b200 -Wl,-rpath,${SRCDIR}/..
#include "simdjson_b200.h"
*/
import "C"

import (
	"errors"
	"unsafe"
)

// one sj_ctx (CUDA stream + device scratch) per concurrent parse, recycled like the reference
// recycles *ParsedJson internals (simdjson_amd64.go:46-51).  A bounded free list, not a sync.Pool:
// a context owns a CUDA stream, events, pinned memory and grow-only device scratch, so a handle
// the pool drops must be destroyed, never just forgotten.
var b200Free = make(chan *C.sj_ctx, 16)

func b200Get() *C.sj_ctx {
	select {
	case h := <-b200Free:
		return h
	default:
	}
	var h *C.sj_ctx
	if rc := C.sj_ctx_create(-1, &h); rc != C.SJ_OK {
		return nil
	}
	return h
}

func b200Put(h *C.sj_ctx) {
	select {
	case b200Free <- h:
	default:
		C.sj_ctx_destroy(h) // more contexts in flight than the list keeps: release the device resources now
	}
}

// SupportedCPU reports whether the GPU path can run (simdjson_amd64.go:37).
func SupportedCPU() bool { return C.sj_supported() != 0 }

func (pj *internalParsedJson) parseMessage(msg []byte, ndjson bool) error {
	h := b200Get()
	if h == nil {
		return errors.New("Host CPU does not meet target specs") // simdjson_amd64.go:43
	}
	defer b200Put(h)

	var flags C.uint32_t
	if ndjson {
		flags |= C.SJ_FLAG_NDJSON
	}
	if pj.copyStrings {
		flags |= C.SJ_FLAG_COPY_STRINGS
	}
	// Output buffers: sj_bounds() is the safe bound (16 bytes of tape per input byte) -- far more than any real
	// document needs, so start from what is there (or an estimate in the spirit of parse_json_amd64.go:30) and
	// let SJ_ERR_CAPACITY, which reports the exact sizes before anything is written, drive one retry.
	if cap(pj.Tape) == 0 {
		pj.Tape = make([]uint64, 0, len(msg)/4+1024)
	}
	if pj.Strings == nil {
		pj.Strings = &TStrings{make([]byte, 0, len(msg)+64)}
	}
	var tapeLen, strLen, off, n C.size_t
	var p *C.uint8_t
	if len(msg) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&msg[0]))
	}
	var tape []uint64
	var strs []byte
	var rc C.int
	for attempt := 0; attempt < 2; attempt++ {
		tape = pj.Tape[:cap(pj.Tape)]
		strs = pj.Strings.B[:cap(pj.Strings.B)]
		rc = C.sj_parse(h, p, C.size_t(len(msg)), flags,
			(*C.uint64_t)(unsafe.Pointer(unsafe.SliceData(tape))), C.size_t(len(tape)), &tapeLen,
			(*C.uint8_t)(unsafe.Pointer(unsafe.SliceData(strs))), C.size_t(len(strs)), &strLen,
			&off, &n)
		if rc != C.SJ_ERR_CAPACITY {
			break
		}
		if int(tapeLen) > cap(pj.Tape) {
			pj.Tape = make([]uint64, 0, int(tapeLen)+int(tapeLen)/8)
		}
		if int(strLen) > cap(pj.Strings.B) {
			pj.Strings.B = make([]byte, 0, int(strLen)+int(strLen)/8+64)
		}
	}
	pj.Message = msg[off : off+n] // bytes.TrimSpace window (parse_json_amd64.go:55)
	switch rc {
	case C.SJ_OK:
		pj.Tape = tape[:tapeLen]
		pj.Strings.B = strs[:strLen]
		pj.isvalid = true
		return nil
	case C.SJ_ERR_STAGE1:
		return errors.New("Failed to find all structural indices for stage 1") // parse_json_amd64.go:93
	case C.SJ_ERR_STAGE2:
		return errors.New("Bad parsing while executing stage 2") // parse_json_amd64.go:81
	default:
		return errors.New(C.GoString(C.sj_error_string(rc)))
	}
}

// ParseAndCountWhere runs parseMessage and the reference's countWhere(key, value, pj)
// (ndjson_test.go:421-459, Object.FindKey parsed_object.go:97-140) in one call with the tape
// left in device memory: records = number of root elements (countObjects, ndjson_test.go:461),
// matches = roots whose object has `key` as a string member equal to `value`.  Only the two
// counts cross PCIe, so the call is bound by the upload of msg, not by the download of a tape
// 1.7x its size.  This is an addition next to the drop-in path, not a replacement of it.
func ParseAndCountWhere(msg []byte, ndjson bool, key, value string) (records, matches uint64, err error) {
	h := b200Get()
	if h == nil {
		return 0, 0, errors.New("Host CPU does not meet target specs")
	}
	defer b200Put(h)
	flags := C.uint32_t(C.SJ_FLAG_COPY_STRINGS)
	if ndjson {
		flags |= C.SJ_FLAG_NDJSON
	}
	var p *C.uint8_t
	if len(msg) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&msg[0]))
	}
	k, v := []byte(key), []byte(value)
	var r, m C.uint64_t
	rc := C.sj_parse_count_where(h, p, C.size_t(len(msg)), flags,
		(*C.uint8_t)(unsafe.Pointer(unsafe.SliceData(k))), C.size_t(len(k)),
		(*C.uint8_t)(unsafe.Pointer(unsafe.SliceData(v))), C.size_t(len(v)), &r, &m)
	switch rc {
	case C.SJ_OK:
		return uint64(r), uint64(m), nil
	case C.SJ_ERR_STAGE1:
		return 0, 0, errors.New("Failed to find all structural indices for stage 1")
	case C.SJ_ERR_STAGE2:
		return 0, 0, errors.New("Bad parsing while executing stage 2")
	default:
		return 0, 0, errors.New(C.GoString(C.sj_error_string(rc)))
	}
}

// ParseAndMarshalJSON runs parseMessage and Iter.MarshalJSON (parsed_json.go:394-556) of the
// whole tape in one call, with the tape left in device memory: the result is the compact JSON
// text, one line per root, byte for byte what pj.Iter().MarshalJSON() returns.  Only the text
// crosses PCIe.  The first attempt uses a buffer of len(msg)+64 bytes; if the text is longer,
// the call is repeated once with the exact size it reported.
func ParseAndMarshalJSON(msg []byte, ndjson bool) ([]byte, error) {
	h := b200Get()
	if h == nil {
		return nil, errors.New("Host CPU does not meet target specs")
	}
	defer b200Put(h)
	flags := C.uint32_t(C.SJ_FLAG_COPY_STRINGS)
	if ndjson {
		flags |= C.SJ_FLAG_NDJSON
	}
	var p *C.uint8_t
	if len(msg) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&msg[0]))
	}
	out := make([]byte, len(msg)+64)
	var n C.size_t
	rc := C.sj_parse_marshal(h, p, C.size_t(len(msg)), flags, (*C.uint8_t)(unsafe.Pointer(&out[0])), C.size_t(len(out)), &n)
	if rc == C.SJ_ERR_CAPACITY {
		out = make([]byte, int(n)+1)
		rc = C.sj_parse_marshal(h, p, C.size_t(len(msg)), flags, (*C.uint8_t)(unsafe.Pointer(&out[0])), C.size_t(len(out)), &n)
	}
	switch rc {
	case C.SJ_OK:
		return out[:int(n)], nil
	case C.SJ_ERR_STAGE1:
		return nil, errors.New("Failed to find all structural indices for stage 1")
	case C.SJ_ERR_STAGE2:
		return nil, errors.New("Bad parsing while executing stage 2")
	default:
		return nil, errors.New(C.GoString(C.sj_error_string(rc)))
	}
}

// ParseAndSerialize runs parseMessage and Serializer.Serialize (parsed_serialize.go:200-431) in
// one call, with the tape left in device memory: the result is the v3 stream with uncompressed
// blocks (CompressNone), which the reference's NewSerializer().Deserialize reads.  Strings are
// deduplicated exactly, keeping the first occurrence, so the stream does not depend on the run or
// on WithCopyStrings.  Only the stream crosses PCIe.  The first attempt uses a buffer of
// 2*len(msg)+64 bytes; if the stream is longer, the call is repeated once at the exact size.
func ParseAndSerialize(msg []byte, ndjson bool) ([]byte, error) {
	h := b200Get()
	if h == nil {
		return nil, errors.New("Host CPU does not meet target specs")
	}
	defer b200Put(h)
	flags := C.uint32_t(C.SJ_FLAG_COPY_STRINGS)
	if ndjson {
		flags |= C.SJ_FLAG_NDJSON
	}
	var p *C.uint8_t
	if len(msg) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&msg[0]))
	}
	out := make([]byte, 2*len(msg)+64)
	var n C.size_t
	rc := C.sj_parse_serialize(h, p, C.size_t(len(msg)), flags, (*C.uint8_t)(unsafe.Pointer(&out[0])), C.size_t(len(out)), &n)
	if rc == C.SJ_ERR_CAPACITY {
		out = make([]byte, int(n)+1)
		rc = C.sj_parse_serialize(h, p, C.size_t(len(msg)), flags, (*C.uint8_t)(unsafe.Pointer(&out[0])), C.size_t(len(out)), &n)
	}
	switch rc {
	case C.SJ_OK:
		return out[:int(n)], nil
	case C.SJ_ERR_STAGE1:
		return nil, errors.New("Failed to find all structural indices for stage 1")
	case C.SJ_ERR_STAGE2:
		return nil, errors.New("Bad parsing while executing stage 2")
	default:
		return nil, errors.New(C.GoString(C.sj_error_string(rc)))
	}
}
