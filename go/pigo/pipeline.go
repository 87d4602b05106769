// pipeline.go -- additive: the face -> ClusterDetections -> pupils -> landmarks sequence of cmd/pigo/main.go:369-565 /
// core/flploc_test.go:75-154 for a whole frame batch, or for images of different sizes, in ONE library call
// (pigo_detect_batch / pigo_detect_images: sequenced on the device).
package pigo

/*
#include <stdlib.h>
#include "pigo_b200.h"
*/
import "C"

import (
	"sync/atomic"
	"unsafe"
)

// LandmarkCall is one GetLandmarkPoint call of the per-face sequence.
type LandmarkCall struct {
	Cascade *PuplocCascade
	FlipV   bool
}

// ReferenceLandmarkCalls returns the reference's 15-call sequence (core/flploc_test.go:122-146, cmd/pigo/main.go:493-563).
func ReferenceLandmarkCalls(flpcs map[string][]*FlpCascade) []LandmarkCall {
	var calls []LandmarkCall
	for _, eye := range []string{"lp46", "lp44", "lp42", "lp38", "lp312"} {
		for _, flpc := range flpcs[eye] {
			calls = append(calls, LandmarkCall{flpc.PuplocCascade, false}, LandmarkCall{flpc.PuplocCascade, true})
		}
	}
	for _, mouth := range []string{"lp93", "lp84", "lp82", "lp81"} {
		for _, flpc := range flpcs[mouth] {
			calls = append(calls, LandmarkCall{flpc.PuplocCascade, false})
		}
	}
	return append(calls, LandmarkCall{flpcs["lp84"][0].PuplocCascade, true})
}

// FaceResult is one clustered face with its refinements (nil / empty when Scale <= MinFaceScale).
type FaceResult struct {
	Face      Detection
	LeftEye   *Puploc
	RightEye  *Puploc
	Landmarks []Puploc
}

// PipelineParams are the knobs the reference's callers hard-code (main.go:404,420; flploc_test.go:102,107).
type PipelineParams struct {
	IoU          float64
	Angle        float64
	MinFaceScale int
	EyePerturbs  int
	FlpPerturbs  int
	Sharded      bool // spread the frames over the GPUs of InitDevices
}

// DetectBatch runs the whole sequence for every frame; result[f] lists frame f's clusters in the reference's order.
func (pg *Pigo) DetectBatch(plc *PuplocCascade, calls []LandmarkCall, frames [][]uint8, cp CascadeParams, pp PipelineParams) [][]FaceResult {
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
	ncalls := len(calls)
	hs, fl := callArrays(calls)
	defer C.free(unsafe.Pointer(hs))
	prm := C.pigo_pipeline_params{min_size: C.int32_t(cp.MinSize), max_size: C.int32_t(cp.MaxSize), shift_factor: C.double(cp.ShiftFactor),
		scale_factor: C.double(cp.ScaleFactor), angle: C.double(pp.Angle), iou_threshold: C.double(pp.IoU),
		min_face_scale: C.int32_t(pp.MinFaceScale), eye_perturbs: C.int32_t(pp.EyePerturbs), flp_perturbs: C.int32_t(pp.FlpPerturbs)}
	key := atomic.AddUint64(&plc.seed, 1)
	faceCap := 32
	for {
		faces := make([]C.pigo_det, nf*faceCap)
		nfaces := make([]C.int, nf)
		points := make([]C.pigo_point, nf*faceCap*(2+ncalls))
		rc, err := call(func() C.int {
			if pp.Sharded {
				return C.pigo_detect_batch_sharded(pg.h, plc.h, hs, &fl[0], C.int(ncalls), (*C.uint8_t)(pinned), C.int(nf),
					C.size_t(stride), C.int(cp.Rows), C.int(cp.Cols), C.int(cp.Dim), &prm, nil, C.uint64_t(key), &faces[0], C.int(faceCap), &nfaces[0], &points[0])
			}
			return C.pigo_detect_batch(pg.h, plc.h, hs, &fl[0], C.int(ncalls), (*C.uint8_t)(pinned), C.int(nf),
				C.size_t(stride), C.int(cp.Rows), C.int(cp.Cols), C.int(cp.Dim), &prm, nil, C.uint64_t(key), &faces[0], C.int(faceCap), &nfaces[0], &points[0],
				C.PIGO_MEM_HOST, nil)
		})
		if rc == C.PIGO_E_CAP {
			grown := false
			for _, n := range nfaces {
				if int(n) > faceCap {
					faceCap, grown = int(n), true
				}
			}
			if !grown {
				prm.det_cap = 4 * (prm.det_cap + 512) // raw detections per frame exceeded det_cap
			}
			continue
		}
		if err != nil {
			panic(err)
		}
		return faceResults(faces, nfaces, points, faceCap, ncalls, pp.MinFaceScale)
	}
}

// callArrays returns the call list as C arrays (cgo: no Go pointers to Go pointers); the caller frees the handle array.
func callArrays(calls []LandmarkCall) (**C.pigo_puploc, []C.uint8_t) {
	hs := unsafe.Slice((**C.pigo_puploc)(C.malloc(C.size_t(len(calls)+1)*C.size_t(unsafe.Sizeof(uintptr(0))))), len(calls)+1)
	fl := make([]C.uint8_t, len(calls)+1)
	for i, c := range calls {
		hs[i] = c.Cascade.h
		if c.FlipV {
			fl[i] = 1
		}
	}
	return &hs[0], fl
}

// faceResults converts the [n][faceCap] faces and [n][faceCap][2+ncalls] points of a pipeline call.
func faceResults(faces []C.pigo_det, nfaces []C.int, points []C.pigo_point, faceCap, ncalls, minFaceScale int) [][]FaceResult {
	out := make([][]FaceResult, len(nfaces))
	for f := range out {
		for k := 0; k < int(nfaces[f]); k++ {
			d := faces[f*faceCap+k]
			fr := FaceResult{Face: Detection{int(d.row), int(d.col), int(d.scale), float32(d.q)}}
			if int(d.scale) > minFaceScale {
				p := points[(f*faceCap+k)*(2+ncalls):]
				fr.LeftEye = &Puploc{Row: int(p[0].row), Col: int(p[0].col), Scale: float32(p[0].scale)}
				fr.RightEye = &Puploc{Row: int(p[1].row), Col: int(p[1].col), Scale: float32(p[1].scale)}
				for c := 0; c < ncalls; c++ {
					fr.Landmarks = append(fr.Landmarks, Puploc{Row: int(p[2+c].row), Col: int(p[2+c].col), Scale: float32(p[2+c].scale)})
				}
			}
			out[f] = append(out[f], fr)
		}
	}
	return out
}

// DetectImages runs the whole sequence for images of different sizes in one call (pigo_detect_images); result[i] lists
// image i's clusters in the reference's order.  cp's MinSize, MaxSize, ShiftFactor and ScaleFactor are shared by every image
// (cp's own ImageParams is not used).  With pp.Sharded the images are spread over the GPUs of InitDevices
// (pigo_detect_images_sharded) in contiguous shards of about equal modelled cost; the result is the same.
func (pg *Pigo) DetectImages(plc *PuplocCascade, calls []LandmarkCall, images []ImageParams, cp CascadeParams, pp PipelineParams) [][]FaceResult {
	n := len(images)
	if n == 0 {
		return nil
	}
	// pixels in one pinned buffer (256-byte aligned slices), descriptors in C memory, as RunCascadeImages does
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
	ncalls := len(calls)
	hs, fl := callArrays(calls)
	defer C.free(unsafe.Pointer(hs))
	prm := C.pigo_pipeline_params{min_size: C.int32_t(cp.MinSize), max_size: C.int32_t(cp.MaxSize), shift_factor: C.double(cp.ShiftFactor),
		scale_factor: C.double(cp.ScaleFactor), angle: C.double(pp.Angle), iou_threshold: C.double(pp.IoU),
		min_face_scale: C.int32_t(pp.MinFaceScale), eye_perturbs: C.int32_t(pp.EyePerturbs), flp_perturbs: C.int32_t(pp.FlpPerturbs)}
	key := atomic.AddUint64(&plc.seed, 1)
	faceCap := 32
	for {
		faces := make([]C.pigo_det, n*faceCap)
		nfaces := make([]C.int, n)
		points := make([]C.pigo_point, n*faceCap*(2+ncalls))
		rc, err := call(func() C.int {
			if pp.Sharded {
				return C.pigo_detect_images_sharded(pg.h, plc.h, hs, &fl[0], C.int(ncalls), &desc[0], C.int(n), nil, &prm, nil, C.uint64_t(key),
					&faces[0], C.int(faceCap), &nfaces[0], &points[0])
			}
			return C.pigo_detect_images(pg.h, plc.h, hs, &fl[0], C.int(ncalls), &desc[0], C.int(n), &prm, nil, C.uint64_t(key), &faces[0],
				C.int(faceCap), &nfaces[0], &points[0], C.PIGO_MEM_HOST, nil)
		})
		if rc == C.PIGO_E_CAP {
			grown := false
			for _, c := range nfaces {
				if int(c) > faceCap {
					faceCap, grown = int(c), true
				}
			}
			if !grown {
				prm.det_cap = 4 * (prm.det_cap + 512) // raw detections per image exceeded det_cap
			}
			continue
		}
		if err != nil {
			panic(err)
		}
		return faceResults(faces, nfaces, points, faceCap, ncalls, pp.MinFaceScale)
	}
}

// DetectImagesAngles is DetectImages with image i scanned and its eyes refined at angles[i] (pigo_detect_images_angles);
// pp.Angle is not used and the landmark calls stay at angle 0, as GetLandmarkPoint does.  A pixel slice listed several
// times (an angle sweep) is copied once (once per device with pp.Sharded, which spreads the images over the GPUs of
// InitDevices like DetectImages).  It panics unless there is one angle per image.
func (pg *Pigo) DetectImagesAngles(plc *PuplocCascade, calls []LandmarkCall, images []ImageParams, cp CascadeParams, pp PipelineParams, angles []float64) [][]FaceResult {
	if len(angles) != len(images) {
		panic("pigo: DetectImagesAngles needs one angle per image")
	}
	n := len(images)
	if n == 0 {
		return nil
	}
	desc, free := packImages(images)
	defer free()
	ncalls := len(calls)
	hs, fl := callArrays(calls)
	defer C.free(unsafe.Pointer(hs))
	prm := C.pigo_pipeline_params{min_size: C.int32_t(cp.MinSize), max_size: C.int32_t(cp.MaxSize), shift_factor: C.double(cp.ShiftFactor),
		scale_factor: C.double(cp.ScaleFactor), iou_threshold: C.double(pp.IoU), min_face_scale: C.int32_t(pp.MinFaceScale),
		eye_perturbs: C.int32_t(pp.EyePerturbs), flp_perturbs: C.int32_t(pp.FlpPerturbs)}
	key := atomic.AddUint64(&plc.seed, 1)
	faceCap := 32
	for {
		faces := make([]C.pigo_det, n*faceCap)
		nfaces := make([]C.int, n)
		points := make([]C.pigo_point, n*faceCap*(2+ncalls))
		rc, err := call(func() C.int {
			if pp.Sharded {
				return C.pigo_detect_images_sharded(pg.h, plc.h, hs, &fl[0], C.int(ncalls), &desc[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])),
					&prm, nil, C.uint64_t(key), &faces[0], C.int(faceCap), &nfaces[0], &points[0])
			}
			return C.pigo_detect_images_angles(pg.h, plc.h, hs, &fl[0], C.int(ncalls), &desc[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])),
				&prm, nil, C.uint64_t(key), &faces[0], C.int(faceCap), &nfaces[0], &points[0], C.PIGO_MEM_HOST, nil)
		})
		if rc == C.PIGO_E_CAP {
			grown := false
			for _, c := range nfaces {
				if int(c) > faceCap {
					faceCap, grown = int(c), true
				}
			}
			if !grown {
				prm.det_cap = 4 * (prm.det_cap + 512) // raw detections per image exceeded det_cap
			}
			continue
		}
		if err != nil {
			panic(err)
		}
		return faceResults(faces, nfaces, points, faceCap, ncalls, pp.MinFaceScale)
	}
}

// SweepFace is one merged face of DetectImagesSweep and the angle it was found at (the value the caller listed); its eyes
// were refined at that angle.
type SweepFace struct {
	FaceResult
	Angle float64
}

// DetectImagesSweep scans every image at every angle of angles, merges each image's lists as RunCascadeImagesSweep does
// (pp.IoU) and refines every merged face with its eyes at its own angle (pigo_detect_images_sweep); pp.Angle and
// pp.Sharded are not used and the landmark calls stay at angle 0, as GetLandmarkPoint does.
func (pg *Pigo) DetectImagesSweep(plc *PuplocCascade, calls []LandmarkCall, images []ImageParams, cp CascadeParams, pp PipelineParams, angles []float64) [][]SweepFace {
	n := len(images)
	if n == 0 || len(angles) == 0 {
		return make([][]SweepFace, n)
	}
	desc, free := packImages(images)
	defer free()
	ncalls := len(calls)
	hs, fl := callArrays(calls)
	defer C.free(unsafe.Pointer(hs))
	prm := C.pigo_pipeline_params{min_size: C.int32_t(cp.MinSize), max_size: C.int32_t(cp.MaxSize), shift_factor: C.double(cp.ShiftFactor),
		scale_factor: C.double(cp.ScaleFactor), iou_threshold: C.double(pp.IoU), min_face_scale: C.int32_t(pp.MinFaceScale),
		eye_perturbs: C.int32_t(pp.EyePerturbs), flp_perturbs: C.int32_t(pp.FlpPerturbs)}
	key := atomic.AddUint64(&plc.seed, 1)
	faceCap := 32
	for {
		faces := make([]C.pigo_det, n*faceCap)
		fangle := make([]C.int32_t, n*faceCap)
		nfaces := make([]C.int, n)
		points := make([]C.pigo_point, n*faceCap*(2+ncalls))
		rc, err := call(func() C.int {
			return C.pigo_detect_images_sweep(pg.h, plc.h, hs, &fl[0], C.int(ncalls), &desc[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])),
				C.int(len(angles)), &prm, nil, C.uint64_t(key), &faces[0], &fangle[0], C.int(faceCap), &nfaces[0], &points[0], C.PIGO_MEM_HOST, nil)
		})
		if rc == C.PIGO_E_CAP {
			grown := false
			for _, c := range nfaces {
				if int(c) > faceCap {
					faceCap, grown = int(c), true
				}
			}
			if !grown {
				prm.det_cap = 4 * (prm.det_cap + 512) // raw detections of an (image, angle) entry exceeded det_cap
			}
			continue
		}
		if err != nil {
			panic(err)
		}
		res := faceResults(faces, nfaces, points, faceCap, ncalls, pp.MinFaceScale)
		out := make([][]SweepFace, n)
		for i := range res {
			for k, fr := range res[i] {
				out[i] = append(out[i], SweepFace{fr, angles[int(fangle[i*faceCap+k])]})
			}
		}
		return out
	}
}
