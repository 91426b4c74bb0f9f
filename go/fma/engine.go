// Package fma is the cgo binding of the H100 sleep/wake weight-movement engine (include/fma_engine.h).
//
// NOT COMPILED OR TESTED IN THIS REPOSITORY'S CI: the build image has no Go toolchain (SURVEY.md §0).  It is the
// reference-side binding a maintainer of llm-d-fast-model-actuation would add for a Go-hosted engine owner
// (north_star: "host code in Go calling CUDA through a thin cgo C-ABI"); the same source is shown in INTEGRATION.md §2.
package fma

/*
#cgo CFLAGS:  -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../llm-d-fast-model-actuation_b200 -lfma_b200 -Wl,-rpath,${SRCDIR}/../../llm-d-fast-model-actuation_b200
#include <stdlib.h>
#include "fma_engine.h"
*/
import "C"

import (
	"fmt"
	"syscall"
	"unsafe"
)

type Engine struct{ h *C.fma_engine_t }

func lastErr(rc C.int) error { return fmt.Errorf("fma: rc=%d: %s", int(rc), C.GoString(C.fma_last_error())) }

// NewEngine replaces the per-process CuMemAllocator singleton (vllm:device_allocator/cumem.py:118-138).
func NewEngine(device int) (*Engine, error) {
	var h *C.fma_engine_t
	if rc := C.fma_engine_create(C.int(device), nil, &h); rc != 0 {
		return nil, lastErr(rc)
	}
	return &Engine{h}, nil
}

func (e *Engine) Close() { C.fma_engine_destroy(e.h) }

func (e *Engine) Tag(name string) (int, error) {
	cs := C.CString(name)
	defer C.free(unsafe.Pointer(cs))
	id := C.fma_tag_intern(e.h, cs)
	if id < 0 {
		return 0, lastErr(id)
	}
	return int(id), nil
}

func (e *Engine) Alloc(bytes uint64, tag int) (uintptr, error) {
	var p unsafe.Pointer
	if rc := C.fma_alloc(e.h, C.size_t(bytes), C.int(tag), &p); rc != 0 {
		return 0, lastErr(rc)
	}
	return uintptr(p), nil
}

// Sleep == POST /sleep?level=1 when offloadMask has the "weights" bit (pkg/controller/dual-pods/inference-server.go:1329-1339).
func (e *Engine) Sleep(offloadMask uint64, tier int) error {
	if rc := C.fma_sleep(e.h, C.uint64_t(offloadMask), C.int(tier), 0); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// WakeUp == POST /wake_up (inference-server.go:1118-1137); tagMask 0 wakes every tag. Safe to retry.
func (e *Engine) WakeUp(tagMask uint64) error {
	if rc := C.fma_wake(e.h, C.uint64_t(tagMask), 0); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// IsSleeping backs api.SleepState{IsSleeping} (pkg/api/interface.go:129-133).
func (e *Engine) IsSleeping() bool { return C.fma_is_sleeping(e.h) == 1 }

// Swap: D2H of the outgoing model overlapped with H2D of the incoming one (BASELINE config 4).
func Swap(out *Engine, offloadMask uint64, in *Engine, wakeMask uint64) error {
	if rc := C.fma_swap(out.h, C.uint64_t(offloadMask), C.FMA_TIER_HOST, in.h, C.uint64_t(wakeMask), 0); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// SetOption changes one knob of a live engine between operations ("mode", "pack", "chunk_bytes", ...: fma_set_option).
// SetOption("pack", 1) turns on the PACKED host image: bf16 weight pages cross PCIe in a lossless 0.758x code.
func (e *Engine) SetOption(key string, value int64) error {
	cs := C.CString(key)
	defer C.free(unsafe.Pointer(cs))
	if rc := C.fma_set_option(e.h, cs, C.int64_t(value)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// HostReserve pins the host store ahead of the first sleep, off the critical path (the reference pins one buffer per
// segment inside its sleep loop, vllm:device_allocator/cumem.py:204-209).
func (e *Engine) HostReserve(bytes uint64) error {
	if rc := C.fma_host_reserve(e.h, C.size_t(bytes)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// PeerReserve prepares a parking buffer in another GPU's HBM for the NVLink tier (BASELINE config 5).
func (e *Engine) PeerReserve(peerDevice int, bytes uint64) error {
	if rc := C.fma_peer_reserve(e.h, C.int(peerDevice), C.size_t(bytes)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// Free releases one segment (my_free of the pluggable allocator).
func (e *Engine) Free(ptr uintptr) error {
	if rc := C.fma_free(e.h, unsafe.Pointer(ptr)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// CurrentUsage mirrors CuMemAllocator.get_current_usage (cumem.py:310-318): bytes of all live segments.
func (e *Engine) CurrentUsage() uint64 { return uint64(C.fma_current_usage(e.h)) }

// LoadSpan is one byte range of a checkpoint file and the device address it lands at.
type LoadSpan struct {
	FileOffset, Bytes uint64
	Dst               uintptr
}

// LoadFile streams byte ranges of one file into mapped segments through the pinned bounce ring and the copy engines
// (the cold "load_model" path, SURVEY.md §8f-3).
func (e *Engine) LoadFile(path string, spans []LoadSpan) (seconds float64, err error) {
	if len(spans) == 0 {
		return 0, nil
	}
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	cspans := make([]C.fma_load_span_t, len(spans))
	for i, s := range spans {
		cspans[i].file_offset = C.uint64_t(s.FileOffset)
		cspans[i].bytes = C.uint64_t(s.Bytes)
		cspans[i].dst = C.uint64_t(s.Dst)
	}
	var st C.fma_load_stats_t
	if rc := C.fma_load_file(e.h, cs, &cspans[0], C.uint32_t(len(spans)), 0, &st); rc != 0 {
		return 0, lastErr(rc)
	}
	return float64(st.seconds), nil
}

// Stats returns the engine's fma_stats_t as cgo sees it, so every field of include/fma_engine.h is there without a Go copy of
// the struct, resident_bytes (the HBM a sleeping image's resident share holds on this GPU) and prefetched_bytes included.
func (e *Engine) Stats() (C.fma_stats_t, error) {
	var st C.fma_stats_t
	if rc := C.fma_stats(e.h, &st); rc != 0 {
		return st, lastErr(rc)
	}
	return st, nil
}

// ---- round 2: node-level parking buffers, multi-path wake, phase timeline ------------------------------------------

// Parking is a node-level owner's exportable parking buffer in one GPU's HBM (fma_parking_create): the launcher pins an
// instance to its own GPUs (inference_server/launcher/launcher.py:171-187), so the OWNER allocates and instances attach by fd.
type Parking struct {
	Handle uint64
	Fd     int
	Bytes  uint64
}

func ParkingCreate(device int, bytes uint64) (*Parking, error) {
	var h C.uint64_t
	var fd C.int
	if rc := C.fma_parking_create(C.int(device), C.size_t(bytes), &h, &fd); rc != 0 {
		return nil, lastErr(rc)
	}
	var nb C.uint64_t
	var fd2 C.int
	if rc := C.fma_parking_export(h, &fd2, &nb); rc != 0 {
		return nil, lastErr(rc)
	}
	syscall.Close(int(fd2))
	return &Parking{Handle: uint64(h), Fd: int(fd), Bytes: uint64(nb)}, nil
}

// ExportFd returns a fresh descriptor to pass to an instance over a unix socket (SCM_RIGHTS).
func (p *Parking) ExportFd() (int, error) {
	var fd C.int
	if rc := C.fma_parking_export(C.uint64_t(p.Handle), &fd, nil); rc != 0 {
		return -1, lastErr(rc)
	}
	return int(fd), nil
}

func (p *Parking) Destroy() { C.fma_parking_destroy(C.uint64_t(p.Handle)); syscall.Close(p.Fd) }

// PeerAttach makes the owner's buffer this engine's peer-tier store; the buffer's GPU need not be visible to this process.
func (e *Engine) PeerAttach(fd int, bytes uint64) error {
	if rc := C.fma_peer_attach(e.h, C.int(fd), C.size_t(bytes)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// ImageDescribe returns the descriptor of the image sleeping in `tier`; the owner keeps it next to the buffer's fd.
func (e *Engine) ImageDescribe(tier int) ([]byte, error) {
	n := C.fma_image_describe(e.h, C.int(tier), nil, 0)
	if n < 0 {
		return nil, lastErr(n)
	}
	buf := make([]byte, int(n))
	if rc := C.fma_image_describe(e.h, C.int(tier), unsafe.Pointer(&buf[0]), C.size_t(n)); rc < 0 {
		return nil, lastErr(rc)
	}
	return buf, nil
}

// ImageAdoptParked: after PeerAttach, a fresh engine with the same segment sequence becomes "asleep with the parked image".
func (e *Engine) ImageAdoptParked(desc []byte, tagMask uint64) error {
	if rc := C.fma_image_adopt_parked(e.h, unsafe.Pointer(&desc[0]), C.size_t(len(desc)), C.uint64_t(tagMask), 0); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// FlagWriteBehind makes a file-tier SleepFlags (or swap) return once the image is in the engine's host store: a background job
// writes the file and then moves the image to the file tier (Writeback).  Ignored for other tiers.
const FlagWriteBehind = uint32(C.FMA_FLAG_WRITE_BEHIND)

// SleepFlags is Sleep with fma_sleep's flags (FMA_FLAG_VERIFY, FlagWriteBehind, ...).
func (e *Engine) SleepFlags(offloadMask uint64, tier int, flags uint32) error {
	if rc := C.fma_sleep(e.h, C.uint64_t(offloadMask), C.int(tier), C.uint32_t(flags)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// Writeback waits up to timeoutS seconds (0 polls, negative waits until it ends) for the last write-behind job: writing is true,
// with the image bytes not yet written, while it writes; false once it committed, was pre-empted by another call, or none was
// started.  A job whose write failed returns its error once; the image then still sleeps in the host tier.
func (e *Engine) Writeback(timeoutS float64) (writing bool, pendingBytes uint64, err error) {
	var pending C.uint64_t
	rc := C.fma_image_writeback(e.h, C.double(timeoutS), &pending)
	if rc < 0 {
		return false, 0, lastErr(rc)
	}
	return rc == 1, uint64(pending), nil
}

// FileStore names the file the next file-tier sleep (Sleep(mask, C.FMA_TIER_FILE)) writes; "" forgets it.  The caller owns the file.
func (e *Engine) FileStore(path string) error {
	var cs *C.char
	if path != "" {
		cs = C.CString(path)
		defer C.free(unsafe.Pointer(cs))
	}
	if rc := C.fma_file_store(e.h, cs); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// ImageAdoptFile: a fully awake engine with the same segment sequence becomes "asleep in the file tier" with the image in `path`
// (written by a file-tier sleep or by image_save); only the descriptor is read, WakeUp streams the data.
func (e *Engine) ImageAdoptFile(path string, tagMask uint64, flags uint32) error {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	if rc := C.fma_image_adopt_file(e.h, cs, C.uint64_t(tagMask), C.uint32_t(flags)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// ImageFileInfo describes an image file from its descriptor tail alone (fma_image_file_info): no engine and no GPU are needed.
type ImageFileInfo struct {
	ImageBytes  uint64 // stored bytes in front of the descriptor
	WeightBytes uint64 // bytes of the segments the image restores
	Segments    int
	Version     int
	Packed      bool
	Digests     bool // every segment carries a K3 digest
	Tags        []string
}

// ReadImageFileInfo reads what the image file at `path` holds, without an engine.
func ReadImageFileInfo(path string) (ImageFileInfo, error) {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	var out C.fma_image_file_info_t
	if rc := C.fma_image_file_info(cs, &out); rc != 0 {
		return ImageFileInfo{}, lastErr(rc)
	}
	info := ImageFileInfo{ImageBytes: uint64(out.image_bytes), WeightBytes: uint64(out.weight_bytes), Segments: int(out.n_segments),
		Version: int(out.version), Packed: out.packed != 0, Digests: out.digests != 0}
	for i := 0; i < int(out.n_tags); i++ {
		info.Tags = append(info.Tags, C.GoString(&out.tags[i][0]))
	}
	return info, nil
}

// MoveImage moves the sleeping image to `tier` without waking it (host DRAM, a file named by FileStore, a peer's or this GPU's
// parking buffer).  The source store stays allocated until HostRelease / PeerRelease; a source file is never touched.
func (e *Engine) MoveImage(tier int) error {
	if rc := C.fma_image_move(e.h, C.int(tier)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// MoveImageFlags is MoveImage with fma_image_move_flags' flags.  FlagWriteBehind demotes a host-tier image to the file tier behind
// the call: the write-behind job writes the file and commits, Writeback waits for it, and any later call pre-empts it.
func (e *Engine) MoveImageFlags(tier int, flags uint32) error {
	if rc := C.fma_image_move_flags(e.h, C.int(tier), C.uint32_t(flags)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// PrefetchImage copies the tail of the sleeping image, up to `bytes` of stored bytes (rounded down to 2 MiB), from host DRAM or
// its file into this GPU's HBM ahead of a wake, without waking it; the next Wake moves only the rest over the link.  0 frees that
// HBM again.  Stats().prefetched_bytes reports what the copy holds.
func (e *Engine) PrefetchImage(bytes uint64) error {
	if rc := C.fma_image_prefetch(e.h, C.uint64_t(bytes)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// VerifyImage checks the sleeping image against the digests it carries, where it lies, without waking it.  It returns the indices
// of the segments whose stored bytes do not match (empty: intact).
func (e *Engine) VerifyImage() ([]int, error) {
	n := int(C.fma_segment_count(e.h))
	if n < 0 {
		return nil, lastErr(C.int(n))
	}
	buf := make([]C.int, n+1)
	rc := C.fma_image_verify(e.h, &buf[0], C.int(n))
	if rc < 0 {
		return nil, lastErr(rc)
	}
	bad := make([]int, 0, int(rc))
	for i := 0; i < int(rc) && i < n; i++ {
		bad = append(bad, int(buf[i]))
	}
	return bad, nil
}

// PathsSet names idle peer GPUs whose PCIe links a host-tier wake may borrow (MULTI-PATH wake); nil turns it off.
func (e *Engine) PathsSet(helpers []int, slotBytes uint64, slots int) error {
	var p *C.int
	c := make([]C.int, len(helpers))
	for i, d := range helpers {
		c[i] = C.int(d)
	}
	if len(c) > 0 {
		p = &c[0]
	}
	if rc := C.fma_paths_set(e.h, p, C.int(len(c)), C.size_t(slotBytes), C.int(slots)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// Timeline returns the per-phase timeline of the last sleep / wake ("op,kind,idx,t0_ms,t1_ms,bytes" lines).
func (e *Engine) Timeline() (string, error) {
	n := C.fma_timeline(e.h, nil, 0)
	if n < 0 {
		return "", lastErr(n)
	}
	buf := make([]byte, int(n)+1)
	if rc := C.fma_timeline(e.h, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf))); rc < 0 {
		return "", lastErr(rc)
	}
	return string(buf[:n]), nil
}

// ---- multi-path wake across processes (the instance cannot see the helper GPUs; the node-level owner drives them) ----

// HelperOpen (owner side): a staging buffer in one helper GPU's HBM; fd goes to the instance (PathsAttach).
func HelperOpen(device int, slotBytes uint64, slots int) (handle uint64, fd int, err error) {
	var h C.uint64_t
	var f C.int
	if rc := C.fma_helper_open(C.int(device), C.size_t(slotBytes), C.int(slots), &h, &f); rc != 0 {
		return 0, -1, lastErr(rc)
	}
	return uint64(h), int(f), nil
}

// StoreAttach (owner side): map + pin the instance's memfd host store (Engine.HostStoreShare).
func StoreAttach(fd int) (uint64, error) {
	var h C.uint64_t
	if rc := C.fma_store_attach(C.int(fd), &h); rc != 0 {
		return 0, lastErr(rc)
	}
	return uint64(h), nil
}

// HelperPull (owner side, one goroutine per helper and wake): pull chunks over that helper's link until the path is done.
func HelperPull(helper, store uint64, mailboxFd, pathIndex int, generation uint64, timeoutS float64) error {
	if rc := C.fma_helper_pull(C.uint64_t(helper), C.uint64_t(store), C.int(mailboxFd), C.int(pathIndex), C.uint64_t(generation), C.double(timeoutS)); rc != 0 {
		return lastErr(rc)
	}
	return nil
}

// PathsAttach (instance side): the owner's staging buffers become remote wake paths; returns the mailbox fd to send to the owner.
func (e *Engine) PathsAttach(stagingFds []int, slotBytes uint64, slots int) (int, error) {
	c := make([]C.int, len(stagingFds))
	for i, f := range stagingFds {
		c[i] = C.int(f)
	}
	var mb C.int
	if rc := C.fma_paths_attach(e.h, &c[0], C.int(len(c)), C.size_t(slotBytes), C.int(slots), &mb); rc != 0 {
		return -1, lastErr(rc)
	}
	return int(mb), nil
}

func (e *Engine) PullNextGeneration() uint64 { return uint64(C.fma_pull_next_generation(e.h)) }

func (e *Engine) HostStoreShare() (int, error) {
	var fd C.int
	if rc := C.fma_host_store_share(e.h, &fd); rc != 0 {
		return -1, lastErr(rc)
	}
	return int(fd), nil
}
