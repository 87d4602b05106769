// Package pigo is the cgo shim that makes libpigo_b200.so a drop-in for the detection path of
// github.com/esimov/pigo/core (package name "pigo"): same exported types, methods and argument meaning, host
// code stays in Go, every hot loop runs in hand-written sm_90a CUDA behind the C-ABI of include/pigo_b200.h.
//
// NOT COMPILED IN THE BUILD CONTAINER: that image has no Go toolchain (SURVEY.md section 0: go/gccgo/tinygo
// absent), so this file is the reference-side binding a maintainer adds (INTEGRATION.md), kept beside the
// Python/ctypes mirror (pigo_b200/__init__.py) that the tests and bench.py drive through the same C-ABI.
//
// Build (where Go and the CUDA runtime exist):
//
//	CGO_CFLAGS="-I${REPO}/include" CGO_LDFLAGS="-L${REPO}/pigo_b200/lib -lpigo_b200" go build ./go/pigo
//
// Mapping (reference file:line -> C entry point):
//
//	NewPigo, (*Pigo).Unpack            core/pigo.go:46,:51-110   -> pigo_cascade_create
//	(*Pigo).RunCascade                 core/pigo.go:212-258      -> pigo_run_cascade
//	(*Pigo).ClusterDetections          core/pigo.go:262-308      -> pigo_cluster (sorts the caller's slice in place)
//	(*PuplocCascade).UnpackCascade     core/puploc.go:38-103     -> pigo_puploc_create
//	(*PuplocCascade).RunDetector       core/puploc.go:239-277    -> pigo_puploc_run (library RNG; reference: math/rand)
//	(*PuplocCascade).GetLandmarkPoint  core/flploc.go:36-57      -> pigo_get_landmark_point
//	UnpackFlp, ReadCascadeDir          core/flploc.go:27-33,:60-81 (file I/O stays in Go)
//	RgbToGrayscale                     core/grayscale.go:8-23    -> pigo_rgba_to_gray / pigo_ycbcr_to_nrgba (fused)
//	GetImage, DecodeImage, ImgToNRGBA  core/image.go:13-90       -> Go decode + pigo_ycbcr_to_nrgba for *image.YCbCr (image.go)
//	additive: (*Pigo).RunCascadeBatch, RunCascadeBatchSharded, DetectBatch, InitDevices, (*Pigo).Close, (*PuplocCascade).Close;
//	          wire.go: the CLI's JSON wire format (cmd/pigo/main.go:88-100)
package pigo

/*
#cgo LDFLAGS: -lpigo_b200
#include <stdlib.h>
#include "pigo_b200.h"
*/
import "C"

import (
	"errors"
	"os"
	"path/filepath"
	"runtime"
	"sync/atomic"
	"unsafe"
)

// CascadeParams mirrors core/pigo.go:16-22.
type CascadeParams struct {
	ImageParams
	MinSize     int
	MaxSize     int
	ShiftFactor float64
	ScaleFactor float64
}

// ImageParams mirrors core/pigo.go:29-34.
type ImageParams struct {
	Pixels []uint8
	Rows   int
	Cols   int
	Dim    int
}

// Detection mirrors core/pigo.go:195-200.
type Detection struct {
	Row   int
	Col   int
	Scale int
	Q     float32
}

// Pigo mirrors core/pigo.go:37-43; the tree tables live on the device behind the handle.
type Pigo struct {
	h *C.pigo_cascade
}

// pigo_last_error() is thread-local in the library and a goroutine may migrate between OS threads between two cgo calls:
// every failing call and the fetch of its message are therefore bracketed by runtime.LockOSThread (ADVICE round 1).
func call(f func() C.int) (C.int, error) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	rc := f()
	if rc == C.PIGO_OK {
		return rc, nil
	}
	return rc, errors.New(C.GoString(C.pigo_last_error()))
}

// InitDevices selects the GPUs of the *Sharded entry points (bit d of mask = device d); additive.
func InitDevices(mask uint) error {
	_, err := call(func() C.int { return C.pigo_init_devices(C.uint(mask)) })
	return err
}

// NewPigo mirrors core/pigo.go:46.
func NewPigo() *Pigo { return &Pigo{} }

// Unpack mirrors core/pigo.go:51-110.  The reference never returns an error and panics on a short packet;
// the shim returns the library's PIGO_E_INVALID as an error instead.
func (pg *Pigo) Unpack(packet []byte) (*Pigo, error) {
	if len(packet) == 0 {
		return nil, errors.New("pigo: empty cascade packet")
	}
	var h *C.pigo_cascade
	if _, err := call(func() C.int {
		return C.pigo_cascade_create((*C.uint8_t)(unsafe.Pointer(&packet[0])), C.size_t(len(packet)), &h)
	}); err != nil {
		return nil, err
	}
	p := &Pigo{h: h}
	runtime.SetFinalizer(p, func(q *Pigo) { q.Close() })
	return p, nil
}

// Close releases the device tables (additive; the reference relies on the GC).
func (pg *Pigo) Close() {
	if pg.h != nil {
		C.pigo_cascade_destroy(pg.h)
		pg.h = nil
	}
}

func toGo(buf []C.pigo_det, n int) []Detection {
	if n == 0 {
		return nil // the reference returns a nil slice when nothing is found (core/pigo.go:257)
	}
	out := make([]Detection, n)
	for i := 0; i < n; i++ {
		out[i] = Detection{int(buf[i].row), int(buf[i].col), int(buf[i].scale), float32(buf[i].q)}
	}
	return out
}

// RunCascade mirrors core/pigo.go:212-258.  The reference has no error path: failures panic, like its
// out-of-range slice accesses would.
func (pg *Pigo) RunCascade(cp CascadeParams, angle float64) []Detection {
	if len(cp.Pixels) == 0 {
		return nil
	}
	capacity := 1024
	for {
		buf := make([]C.pigo_det, capacity)
		var n C.int
		rc, err := call(func() C.int {
			return C.pigo_run_cascade(pg.h, (*C.uint8_t)(unsafe.Pointer(&cp.Pixels[0])), C.int(cp.Rows), C.int(cp.Cols), C.int(cp.Dim),
				C.int(cp.MinSize), C.int(cp.MaxSize), C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), C.double(angle),
				&buf[0], C.int(capacity), &n)
		})
		if rc == C.PIGO_E_CAP {
			capacity = int(n)
			continue
		}
		if err != nil {
			panic(err)
		}
		return toGo(buf, int(n))
	}
}

// RunCascadeBatch is additive: frames of identical geometry, one []Detection per frame.
func (pg *Pigo) RunCascadeBatch(frames [][]uint8, cp CascadeParams, angle float64) [][]Detection {
	return pg.runBatch(frames, cp, angle, false)
}

// RunCascadeBatchSharded is RunCascadeBatch over the GPUs selected with InitDevices (frames sharded contiguously, identical result).
func (pg *Pigo) RunCascadeBatchSharded(frames [][]uint8, cp CascadeParams, angle float64) [][]Detection {
	return pg.runBatch(frames, cp, angle, true)
}

func (pg *Pigo) runBatch(frames [][]uint8, cp CascadeParams, angle float64, sharded bool) [][]Detection {
	nf := len(frames)
	if nf == 0 {
		return nil
	}
	stride := cp.Rows * cp.Dim
	var pinned unsafe.Pointer
	if _, err := call(func() C.int { return C.pigo_alloc_pinned(&pinned, C.size_t(stride*nf)) }); err != nil {
		panic(err)
	}
	defer C.pigo_free_pinned(pinned)
	host := unsafe.Slice((*uint8)(pinned), stride*nf)
	for i, f := range frames {
		copy(host[i*stride:(i+1)*stride], f)
	}
	capacity := 1024
	for {
		buf := make([]C.pigo_det, capacity*nf)
		cnt := make([]C.int, nf)
		rc, err := call(func() C.int {
			if sharded {
				return C.pigo_run_cascade_batch_sharded(pg.h, (*C.uint8_t)(pinned), C.int(nf), C.size_t(stride), C.int(cp.Rows), C.int(cp.Cols),
					C.int(cp.Dim), C.int(cp.MinSize), C.int(cp.MaxSize), C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), C.double(angle),
					&buf[0], C.int(capacity), &cnt[0])
			}
			return C.pigo_run_cascade_batch(pg.h, (*C.uint8_t)(pinned), C.int(nf), C.size_t(stride), C.int(cp.Rows), C.int(cp.Cols), C.int(cp.Dim),
				C.int(cp.MinSize), C.int(cp.MaxSize), C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), C.double(angle),
				&buf[0], C.int(capacity), &cnt[0], C.PIGO_MEM_HOST, nil)
		})
		if rc == C.PIGO_E_CAP {
			for _, c := range cnt {
				if int(c) > capacity {
					capacity = int(c)
				}
			}
			continue
		}
		if err != nil {
			panic(err)
		}
		out := make([][]Detection, nf)
		for i := range out {
			out[i] = toGo(buf[i*capacity:(i+1)*capacity], int(cnt[i]))
		}
		return out
	}
}

// ClusterDetections mirrors core/pigo.go:262-308, including the in-place sort of the caller's slice by Q.
func (pg *Pigo) ClusterDetections(detections []Detection, iouThreshold float64) []Detection {
	n := len(detections)
	if n == 0 {
		return []Detection{}
	}
	in := make([]C.pigo_det, n)
	for i, d := range detections {
		in[i] = C.pigo_det{row: C.int32_t(d.Row), col: C.int32_t(d.Col), scale: C.int32_t(d.Scale), q: C.float(d.Q)}
	}
	out := make([]C.pigo_det, n)
	var k C.int
	if _, err := call(func() C.int { return C.pigo_cluster(&in[0], C.int(n), C.double(iouThreshold), &out[0], C.int(n), &k) }); err != nil {
		panic(err)
	}
	for i := range detections { // the reference sorts its argument (core/pigo.go:264)
		detections[i] = Detection{int(in[i].row), int(in[i].col), int(in[i].scale), float32(in[i].q)}
	}
	res := toGo(out, int(k))
	if res == nil {
		res = []Detection{}
	}
	return res
}

// Puploc mirrors core/puploc.go:14-19.
type Puploc struct {
	Row      int
	Col      int
	Scale    float32
	Perturbs int
}

// PuplocCascade mirrors core/puploc.go:23-30.
type PuplocCascade struct {
	h *C.pigo_puploc
	// seed keys the library's counter-based generator; the reference draws from the auto-seeded global math/rand
	// (core/puploc.go:248-250) and is therefore not reproducible either.  Bumped atomically: RunDetector is re-entrant on a
	// shared cascade in the reference (sync.Pool scratch, core/puploc.go:228) and stays so here.
	seed uint64
}

// SetSeed fixes the generator key of the next RunDetector / GetLandmarkPoint calls (additive; for reproducible runs).
func (plc *PuplocCascade) SetSeed(s uint64) { atomic.StoreUint64(&plc.seed, s) }

// NewPuplocCascade mirrors core/puploc.go:33.
func NewPuplocCascade() *PuplocCascade { return &PuplocCascade{} }

// UnpackCascade mirrors core/puploc.go:38-103.
func (plc *PuplocCascade) UnpackCascade(packet []byte) (*PuplocCascade, error) {
	if len(packet) == 0 {
		return nil, errors.New("pigo: empty cascade packet")
	}
	var h *C.pigo_puploc
	if _, err := call(func() C.int {
		return C.pigo_puploc_create((*C.uint8_t)(unsafe.Pointer(&packet[0])), C.size_t(len(packet)), &h)
	}); err != nil {
		return nil, err
	}
	p := &PuplocCascade{h: h}
	runtime.SetFinalizer(p, func(q *PuplocCascade) { q.Close() })
	return p, nil
}

// Close releases the device tables (additive).
func (plc *PuplocCascade) Close() {
	if plc.h != nil {
		C.pigo_puploc_destroy(plc.h)
		plc.h = nil
	}
}

// RunDetector mirrors core/puploc.go:239-277.
func (plc *PuplocCascade) RunDetector(pl Puploc, img ImageParams, angle float64, flipV bool) *Puploc {
	seed := C.pigo_point{row: C.int32_t(pl.Row), col: C.int32_t(pl.Col), scale: C.float(pl.Scale), perturbs: C.int32_t(pl.Perturbs)}
	var out C.pigo_point
	var fl C.uint8_t
	if flipV {
		fl = 1
	}
	key := atomic.AddUint64(&plc.seed, 1)
	if _, err := call(func() C.int {
		return C.pigo_puploc_run(plc.h, &seed, 1, nil, C.uint64_t(key), (*C.uint8_t)(unsafe.Pointer(&img.Pixels[0])),
			C.int(img.Rows), C.int(img.Cols), C.int(img.Dim), C.double(angle), &fl, &out, C.PIGO_MEM_HOST, nil)
	}); err != nil {
		panic(err) // e.g. Perturbs > 63: the reference panics with index out of range (core/puploc.go:261)
	}
	return &Puploc{Row: int(out.row), Col: int(out.col), Scale: float32(out.scale)}
}

// GetLandmarkPoint mirrors core/flploc.go:36-57.
func (plc *PuplocCascade) GetLandmarkPoint(leftEye, rightEye *Puploc, img ImageParams, perturb int, flipV bool) *Puploc {
	le := C.pigo_point{row: C.int32_t(leftEye.Row), col: C.int32_t(leftEye.Col), scale: C.float(leftEye.Scale)}
	re := C.pigo_point{row: C.int32_t(rightEye.Row), col: C.int32_t(rightEye.Col), scale: C.float(rightEye.Scale)}
	var out C.pigo_point
	fl := C.int(0)
	if flipV {
		fl = 1
	}
	key := atomic.AddUint64(&plc.seed, 1)
	if _, err := call(func() C.int {
		return C.pigo_get_landmark_point(plc.h, &le, &re, (*C.uint8_t)(unsafe.Pointer(&img.Pixels[0])), C.int(img.Rows), C.int(img.Cols),
			C.int(img.Dim), C.int(perturb), fl, nil, C.uint64_t(key), &out)
	}); err != nil {
		panic(err)
	}
	return &Puploc{Row: int(out.row), Col: int(out.col), Scale: float32(out.scale)}
}

// FlpCascade mirrors core/flploc.go:12-15.
type FlpCascade struct {
	*PuplocCascade
	error
}

// UnpackFlp mirrors core/flploc.go:27-33.
func (plc *PuplocCascade) UnpackFlp(cf string) (*PuplocCascade, error) {
	flpc, err := os.ReadFile(cf)
	if err != nil {
		return nil, err
	}
	return plc.UnpackCascade(flpc)
}

// ReadCascadeDir mirrors core/flploc.go:60-81.
func (plc *PuplocCascade) ReadCascadeDir(path string) (map[string][]*FlpCascade, error) {
	cascades, err := os.ReadDir(path)
	if err != nil {
		return nil, err
	}
	if len(cascades) == 0 {
		return nil, errors.New("the provided directory is empty")
	}
	flpcs := make(map[string][]*FlpCascade, len(cascades))
	for _, cascade := range cascades {
		cf, err := filepath.Abs(path + "/" + cascade.Name())
		if err != nil {
			return nil, err
		}
		flpc, err := plc.UnpackFlp(cf)
		flpcs[cascade.Name()] = append(flpcs[cascade.Name()], &FlpCascade{flpc, err})
	}
	return flpcs, err
}
