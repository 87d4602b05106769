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

// RunCascadeImages is additive: RunCascade for images of different sizes in one call.  Result i is what RunCascade returns
// for images[i] with cp's MinSize, MaxSize, ShiftFactor and ScaleFactor (cp's own ImageParams is not used).
func (pg *Pigo) RunCascadeImages(images []ImageParams, cp CascadeParams, angle float64) [][]Detection {
	n := len(images)
	if n == 0 {
		return nil
	}
	// cgo forbids passing Go memory that holds Go pointers: the pixels go to one pinned buffer (256-byte aligned slices)
	// and the descriptors that point into it to C memory
	offs := make([]int, n)
	total := 0
	for i, im := range images {
		offs[i] = total
		total += (len(im.Pixels) + 255) &^ 255
	}
	var pinned unsafe.Pointer
	if _, err := call(func() C.int { return C.pigo_alloc_pinned(&pinned, C.size_t(total+256)) }); err != nil {
		panic(err)
	}
	defer C.pigo_free_pinned(pinned)
	host := unsafe.Slice((*uint8)(pinned), total+256)
	desc := unsafe.Slice((*C.pigo_image)(C.malloc(C.size_t(n)*C.size_t(unsafe.Sizeof(C.pigo_image{})))), n)
	defer C.free(unsafe.Pointer(&desc[0]))
	for i, im := range images {
		copy(host[offs[i]:], im.Pixels)
		desc[i] = C.pigo_image{pixels: (*C.uint8_t)(unsafe.Pointer(&host[offs[i]])), rows: C.int32_t(im.Rows), cols: C.int32_t(im.Cols),
			dim: C.int32_t(im.Dim)}
	}
	capacity := 1024
	for {
		buf := make([]C.pigo_det, capacity*n)
		cnt := make([]C.int, n)
		rc, err := call(func() C.int {
			return C.pigo_run_cascade_images(pg.h, &desc[0], C.int(n), C.int(cp.MinSize), C.int(cp.MaxSize), C.double(cp.ShiftFactor),
				C.double(cp.ScaleFactor), C.double(angle), &buf[0], C.int(capacity), &cnt[0], C.PIGO_MEM_HOST, nil)
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
		out := make([][]Detection, n)
		for i := range out {
			out[i] = toGo(buf[i*capacity:(i+1)*capacity], int(cnt[i]))
		}
		return out
	}
}

// packImages copies the pixels of a mixed-size call to one pinned buffer (256-byte aligned slices; cgo forbids passing Go
// memory that holds Go pointers) and builds the descriptors that point into it in C memory.  Images that share a pixel
// slice and geometry are stored once: an angle sweep lists one image once per angle.  free releases both buffers.
func packImages(images []ImageParams) (desc []C.pigo_image, free func()) {
	type key struct {
		p                  *uint8
		n, rows, cols, dim int
	}
	n := len(images)
	offs := make([]int, n)
	first := make([]bool, n)
	seen := make(map[key]int, n)
	total := 0
	for i, im := range images {
		k := key{nil, len(im.Pixels), im.Rows, im.Cols, im.Dim}
		if len(im.Pixels) > 0 {
			k.p = &im.Pixels[0]
		}
		o, ok := seen[k]
		if !ok {
			o, first[i] = total, true
			seen[k] = o
			total += (len(im.Pixels) + 255) &^ 255
		}
		offs[i] = o
	}
	var pinned unsafe.Pointer
	if _, err := call(func() C.int { return C.pigo_alloc_pinned(&pinned, C.size_t(total+256)) }); err != nil {
		panic(err)
	}
	host := unsafe.Slice((*uint8)(pinned), total+256)
	desc = unsafe.Slice((*C.pigo_image)(C.malloc(C.size_t(n)*C.size_t(unsafe.Sizeof(C.pigo_image{})))), n)
	for i, im := range images {
		if first[i] {
			copy(host[offs[i]:], im.Pixels)
		}
		desc[i] = C.pigo_image{pixels: (*C.uint8_t)(unsafe.Pointer(&host[offs[i]])), rows: C.int32_t(im.Rows), cols: C.int32_t(im.Cols),
			dim: C.int32_t(im.Dim)}
	}
	return desc, func() {
		C.free(unsafe.Pointer(&desc[0]))
		C.pigo_free_pinned(pinned)
	}
}

// RunCascadeImagesAngles is RunCascadeImages with images[i] scanned at angles[i] (pigo_run_cascade_images_angles): an
// angle sweep is one call that lists an image once per angle, and a pixel slice listed several times is copied once.
// It panics unless there is one angle per image.
func (pg *Pigo) RunCascadeImagesAngles(images []ImageParams, cp CascadeParams, angles []float64) [][]Detection {
	if len(angles) != len(images) {
		panic("pigo: RunCascadeImagesAngles needs one angle per image")
	}
	n := len(images)
	if n == 0 {
		return nil
	}
	desc, free := packImages(images)
	defer free()
	capacity := 1024
	for {
		buf := make([]C.pigo_det, capacity*n)
		cnt := make([]C.int, n)
		rc, err := call(func() C.int {
			return C.pigo_run_cascade_images_angles(pg.h, &desc[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])), C.int(cp.MinSize),
				C.int(cp.MaxSize), C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), &buf[0], C.int(capacity), &cnt[0], C.PIGO_MEM_HOST, nil)
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
		out := make([][]Detection, n)
		for i := range out {
			out[i] = toGo(buf[i*capacity:(i+1)*capacity], int(cnt[i]))
		}
		return out
	}
}

// RunCascadeImagesSharded is RunCascadeImagesAngles over the GPUs of InitDevices (pigo_run_cascade_images_sharded): the
// images are cut into contiguous shards of about equal modelled cost, one per device, and the result equals the single-GPU
// call's.  angles is nil (every image at 0) or has one entry per image; any other length panics.
func (pg *Pigo) RunCascadeImagesSharded(images []ImageParams, cp CascadeParams, angles []float64) [][]Detection {
	n := len(images)
	if angles != nil && len(angles) != n {
		panic("pigo: RunCascadeImagesSharded needs nil angles or one angle per image")
	}
	if n == 0 {
		return nil
	}
	desc, free := packImages(images)
	defer free()
	return runCapped(n, func(buf *C.pigo_det, capacity C.int, cnt *C.int) C.int {
		return C.pigo_run_cascade_images_sharded(pg.h, &desc[0], C.int(n), anglesPtr(angles), C.int(cp.MinSize), C.int(cp.MaxSize),
			C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), buf, capacity, cnt)
	})
}

// RunCascadeImagesParams runs the list of reference calls RunCascade(cps[i], angles[i]) as one call
// (pigo_run_cascade_images_params): each CascadeParams carries its own ImageParams, MinSize, MaxSize, ShiftFactor and
// ScaleFactor, and result[i] is what RunCascade(cps[i], angles[i]) returns.  angles is nil (every image unrotated) or has
// one entry per image; any other length panics.  A pixel slice listed several times is copied once.
func (pg *Pigo) RunCascadeImagesParams(cps []CascadeParams, angles []float64) [][]Detection {
	n := len(cps)
	if angles != nil && len(angles) != n {
		panic("pigo: RunCascadeImagesParams needs nil angles or one angle per image")
	}
	if n == 0 {
		return nil
	}
	images, prm, freePrm := cascadeParams(cps)
	defer freePrm()
	desc, free := packImages(images)
	defer free()
	return runCapped(n, func(buf *C.pigo_det, capacity C.int, cnt *C.int) C.int {
		return C.pigo_run_cascade_images_params(pg.h, &desc[0], C.int(n), &prm[0], anglesPtr(angles), buf, capacity, cnt, C.PIGO_MEM_HOST, nil)
	})
}

// cascadeParams splits cps into their images and their pigo_cascade_params (in C memory); free releases the latter.
func cascadeParams(cps []CascadeParams) (images []ImageParams, prm []C.pigo_cascade_params, free func()) {
	n := len(cps)
	images = make([]ImageParams, n)
	prm = unsafe.Slice((*C.pigo_cascade_params)(C.malloc(C.size_t(n)*C.size_t(unsafe.Sizeof(C.pigo_cascade_params{})))), n)
	for i, cp := range cps {
		images[i] = cp.ImageParams
		prm[i] = C.pigo_cascade_params{min_size: C.int32_t(cp.MinSize), max_size: C.int32_t(cp.MaxSize), shift_factor: C.double(cp.ShiftFactor),
			scale_factor: C.double(cp.ScaleFactor)}
	}
	return images, prm, func() { C.free(unsafe.Pointer(&prm[0])) }
}

// anglesPtr is the C view of angles (nil stays NULL).
func anglesPtr(angles []float64) *C.double {
	if len(angles) == 0 {
		return nil
	}
	return (*C.double)(unsafe.Pointer(&angles[0]))
}

// runCapped calls f(out [n][capacity], capacity, counts [n]) until the capacity is enough (PIGO_E_CAP retries with the
// largest reported count) and returns the detections of every entry.
func runCapped(n int, f func(buf *C.pigo_det, capacity C.int, cnt *C.int) C.int) [][]Detection {
	capacity := 1024
	for {
		buf := make([]C.pigo_det, capacity*n)
		cnt := make([]C.int, n)
		rc, err := call(func() C.int { return f(&buf[0], C.int(capacity), &cnt[0]) })
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
		out := make([][]Detection, n)
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

// SweepDetection is one merged face of an angle sweep and the angle it was found at: Angle is the value the caller listed.
type SweepDetection struct {
	Detection
	Angle float64
}

// RunCascadeImagesSweep scans every image at every angle of angles and merges each image's lists
// (pigo_run_cascade_images_sweep): result[i] is ClusterDetections(iou) of image i's RunCascade lists over the angles,
// concatenated in angle order, each cluster with the listed angle of its largest-Q member.  Listing two values of one
// orientation (0 and 1) counts every face found there twice.  A pixel slice is copied to the device once.
func (pg *Pigo) RunCascadeImagesSweep(images []ImageParams, cp CascadeParams, angles []float64, iou float64) [][]SweepDetection {
	n := len(images)
	if n == 0 || len(angles) == 0 {
		return make([][]SweepDetection, n)
	}
	desc, free := packImages(images)
	defer free()
	capacity, detCap := 64, 0
	for {
		buf := make([]C.pigo_det, capacity*n)
		idx := make([]C.int32_t, capacity*n)
		cnt := make([]C.int, n)
		rc, err := call(func() C.int {
			return C.pigo_run_cascade_images_sweep(pg.h, &desc[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])), C.int(len(angles)),
				C.int(cp.MinSize), C.int(cp.MaxSize), C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), C.double(iou), C.int(detCap), &buf[0],
				&idx[0], C.int(capacity), &cnt[0], C.PIGO_MEM_HOST, nil)
		})
		if rc == C.PIGO_E_CAP {
			grown := false
			for _, c := range cnt {
				if int(c) > capacity {
					capacity, grown = int(c), true
				}
			}
			if !grown {
				detCap = 4 * (detCap + 512) // raw detections of an (image, angle) entry exceeded det_cap
			}
			continue
		}
		if err != nil {
			panic(err)
		}
		out := make([][]SweepDetection, n)
		for i := range out {
			dets := toGo(buf[i*capacity:(i+1)*capacity], int(cnt[i]))
			for k, d := range dets {
				out[i] = append(out[i], SweepDetection{d, angles[int(idx[i*capacity+k])]})
			}
		}
		return out
	}
}
