// decoded.go -- additive: detection straight from decoded images (what image.Decode returns for JPEG and PNG files) of any
// size.  The images are packed once into pinned memory in their own pixel format, converted to the reference's gray buffer
// RgbToGrayscale(ImgToNRGBA(img)) (cmd/pigo/main.go:281-286) by one pigo_gray_images call into device memory, and scanned
// there by the mixed-size calls: 1.5 bytes per pixel cross PCIe for a 4:2:0 JPEG instead of the 11.5 of ImgToNRGBA +
// RgbToGrayscale + DetectImages.
package pigo

/*
#include <stdlib.h>
#include "pigo_b200.h"
*/
import "C"

import (
	"image"
	"image/color"
	"reflect"
	"sync/atomic"
	"unsafe"
)

// decodedPart is one distinct image of a decoded batch: its pigo_decoded fields and the host bytes of each plane, from the
// rectangle's origin to its last sample.
type decodedPart struct {
	format, subsample, minX, minY, width, height int
	planes                                       [3][]uint8
	strides                                      [2]int
}

// partOf describes img in its own pixel format: *image.YCbCr with Rect.Min >= 0, *image.NRGBA, *image.RGBA, *image.Gray,
// *image.Gray16, *image.RGBA64, *image.NRGBA64, *image.CMYK and *image.Paletted with a non-empty palette as they are (every
// type image/jpeg and image/png return); other types (*image.NYCbCrA, *image.Alpha, *image.Alpha16, user types), a YCbCr
// image with a negative origin and an empty palette (which panics like the reference) through the shim's ImgToNRGBA as NRGBA.
func partOf(img image.Image) decodedPart {
	b := img.Bounds()
	w, h := b.Dx(), b.Dy()
	p := decodedPart{minX: b.Min.X, minY: b.Min.Y, width: w, height: h}
	if w <= 0 || h <= 0 {
		return p // the library rejects the empty rectangle
	}
	last := image.Pt(b.Max.X-1, b.Max.Y-1)
	switch src := img.(type) {
	case *image.YCbCr:
		if b.Min.X >= 0 && b.Min.Y >= 0 {
			yo, co := src.YOffset(b.Min.X, b.Min.Y), src.COffset(b.Min.X, b.Min.Y)
			ye, ce := src.YOffset(last.X, last.Y)+1, src.COffset(last.X, last.Y)+1
			p.format, p.subsample = C.PIGO_DECODED_YCBCR, int(src.SubsampleRatio)
			p.planes = [3][]uint8{src.Y[yo:ye], src.Cb[co:ce], src.Cr[co:ce]}
			p.strides = [2]int{src.YStride, src.CStride}
			return p
		}
	case *image.NRGBA:
		p.format, p.planes[0], p.strides[0] = C.PIGO_DECODED_NRGBA, src.Pix[src.PixOffset(b.Min.X, b.Min.Y):src.PixOffset(last.X, last.Y)+4], src.Stride
		p.minX, p.minY = 0, 0
		return p
	case *image.RGBA:
		p.format, p.planes[0], p.strides[0] = C.PIGO_DECODED_RGBA, src.Pix[src.PixOffset(b.Min.X, b.Min.Y):src.PixOffset(last.X, last.Y)+4], src.Stride
		p.minX, p.minY = 0, 0
		return p
	case *image.Gray:
		p.format, p.planes[0], p.strides[0] = C.PIGO_DECODED_GRAY, src.Pix[src.PixOffset(b.Min.X, b.Min.Y):src.PixOffset(last.X, last.Y)+1], src.Stride
		p.minX, p.minY = 0, 0
		return p
	case *image.Gray16:
		p.format, p.planes[0], p.strides[0] = C.PIGO_DECODED_GRAY16, src.Pix[src.PixOffset(b.Min.X, b.Min.Y):src.PixOffset(last.X, last.Y)+2], src.Stride
		p.minX, p.minY = 0, 0
		return p
	case *image.RGBA64:
		p.format, p.planes[0], p.strides[0] = C.PIGO_DECODED_RGBA64, src.Pix[src.PixOffset(b.Min.X, b.Min.Y):src.PixOffset(last.X, last.Y)+8], src.Stride
		p.minX, p.minY = 0, 0
		return p
	case *image.NRGBA64:
		p.format, p.planes[0], p.strides[0] = C.PIGO_DECODED_NRGBA64, src.Pix[src.PixOffset(b.Min.X, b.Min.Y):src.PixOffset(last.X, last.Y)+8], src.Stride
		p.minX, p.minY = 0, 0
		return p
	case *image.CMYK:
		p.format, p.planes[0], p.strides[0] = C.PIGO_DECODED_CMYK, src.Pix[src.PixOffset(b.Min.X, b.Min.Y):src.PixOffset(last.X, last.Y)+4], src.Stride
		p.minX, p.minY = 0, 0
		return p
	case *image.Paletted:
		if len(src.Palette) > 0 {
			// an index is a byte: entries past 255 are unreachable.  Each entry is converted the way ImgToNRGBA converts
			// the pixel that uses it, so the result is exact by construction.
			k := min(len(src.Palette), 256)
			pal := make([]uint8, 4*k)
			for i, c := range src.Palette[:k] {
				n := color.NRGBAModel.Convert(c).(color.NRGBA)
				pal[4*i], pal[4*i+1], pal[4*i+2], pal[4*i+3] = n.R, n.G, n.B, n.A
			}
			p.format = C.PIGO_DECODED_PALETTED
			p.planes = [3][]uint8{src.Pix[src.PixOffset(b.Min.X, b.Min.Y) : src.PixOffset(last.X, last.Y)+1], pal}
			p.strides = [2]int{src.Stride, k}
			p.minX, p.minY = 0, 0
			return p
		}
	}
	n := ImgToNRGBA(img)
	return decodedPart{format: C.PIGO_DECODED_NRGBA, width: w, height: h, planes: [3][]uint8{n.Pix[:(h-1)*n.Stride+4*w]}, strides: [2]int{n.Stride, 0}}
}

// packDecoded copies the planes of every distinct image to one pinned buffer (256-byte aligned) and builds the
// descriptors in C memory; an image listed several times is packed once and gets identical descriptors.
func packDecoded(imgs []image.Image) (desc []C.pigo_decoded, free func()) {
	n := len(imgs)
	index := make([]int, n) // image i uses parts[index[i]]
	var parts []decodedPart
	seen := make(map[interface{}]int, n)
	for i, img := range imgs {
		comparable := img != nil && reflect.TypeOf(img).Comparable()
		if comparable {
			if k, ok := seen[img]; ok {
				index[i] = k
				continue
			}
			seen[img] = len(parts)
		}
		index[i] = len(parts)
		parts = append(parts, partOf(img))
	}
	offs := make([][3]int, len(parts))
	total := 0
	for k, p := range parts {
		for j, pl := range p.planes {
			offs[k][j] = total
			total += (len(pl) + 255) &^ 255
		}
	}
	var pinned unsafe.Pointer
	if _, err := call(func() C.int { return C.pigo_alloc_pinned(&pinned, C.size_t(total+256)) }); err != nil {
		panic(err)
	}
	host := unsafe.Slice((*uint8)(pinned), total+256)
	descs := make([]C.pigo_decoded, len(parts))
	for k, p := range parts {
		d := C.pigo_decoded{format: C.int32_t(p.format), subsample: C.int32_t(p.subsample), min_x: C.int32_t(p.minX), min_y: C.int32_t(p.minY),
			width: C.int32_t(p.width), height: C.int32_t(p.height)}
		for j, pl := range p.planes {
			if len(pl) > 0 {
				copy(host[offs[k][j]:], pl)
				d.plane[j] = (*C.uint8_t)(unsafe.Pointer(&host[offs[k][j]]))
			}
		}
		d.stride[0], d.stride[1] = C.int32_t(p.strides[0]), C.int32_t(p.strides[1])
		descs[k] = d
	}
	desc = unsafe.Slice((*C.pigo_decoded)(C.malloc(C.size_t(n+1)*C.size_t(unsafe.Sizeof(C.pigo_decoded{})))), n+1)
	for i := range imgs {
		desc[i] = descs[index[i]]
	}
	return desc[:n], func() {
		C.free(unsafe.Pointer(&desc[0]))
		C.pigo_free_pinned(pinned)
	}
}

// grayDecoded converts imgs into one device arena (pigo_gray_images) and returns the device image descriptors in C memory;
// free releases the arena and the descriptors.
func grayDecoded(imgs []image.Image) (images []C.pigo_image, free func()) {
	n := len(imgs)
	desc, freeDesc := packDecoded(imgs)
	defer freeDesc() // the host planes are read only during the call
	images = unsafe.Slice((*C.pigo_image)(C.malloc(C.size_t(n)*C.size_t(unsafe.Sizeof(C.pigo_image{})))), n)
	var need C.size_t
	var arena unsafe.Pointer
	for {
		rc, err := call(func() C.int {
			return C.pigo_gray_images(&desc[0], C.int(n), (*C.uint8_t)(arena), &need, &images[0], C.PIGO_MEM_HOST, nil)
		})
		if rc == C.PIGO_E_CAP {
			if arena != nil {
				C.pigo_device_free(arena)
				arena = nil
			}
			if _, err := call(func() C.int { return C.pigo_device_alloc(&arena, need) }); err != nil {
				C.free(unsafe.Pointer(&images[0]))
				panic(err)
			}
			continue
		}
		if err != nil {
			C.free(unsafe.Pointer(&images[0]))
			if arena != nil {
				C.pigo_device_free(arena)
			}
			panic(err)
		}
		return images, func() {
			C.free(unsafe.Pointer(&images[0]))
			C.pigo_device_free(arena)
		}
	}
}

// decodedAngles returns angles, or one 0 per image when angles is nil; any other length panics.
func decodedAngles(fn string, angles []float64, n int) []float64 {
	if angles == nil {
		return make([]float64, n)
	}
	if len(angles) != n {
		panic("pigo: " + fn + " needs nil angles or one angle per image")
	}
	return angles
}

// RunCascadeDecoded runs RunCascade on RgbToGrayscale(ImgToNRGBA(img)) of every decoded image (any size, any image.Image)
// in one conversion and one scan: imgs[i] at angles[i], or at 0 when angles is nil.  cp's MinSize, MaxSize, ShiftFactor and
// ScaleFactor are shared (cp's own ImageParams is not used); result[i] is what RunCascade returns for image i alone.
func (pg *Pigo) RunCascadeDecoded(imgs []image.Image, cp CascadeParams, angles []float64) [][]Detection {
	n := len(imgs)
	angles = decodedAngles("RunCascadeDecoded", angles, n)
	if n == 0 {
		return nil
	}
	images, free := grayDecoded(imgs)
	defer free()
	capacity := 1024
	for {
		buf := make([]C.pigo_det, capacity*n)
		cnt := make([]C.int, n)
		rc, err := call(func() C.int {
			return C.pigo_run_cascade_images_angles(pg.h, &images[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])), C.int(cp.MinSize),
				C.int(cp.MaxSize), C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), &buf[0], C.int(capacity), &cnt[0], C.PIGO_FRAMES_DEVICE, nil)
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

// RunCascadeDecodedSharded is RunCascadeDecoded over the GPUs of InitDevices (pigo_run_cascade_decoded_sharded): the
// images, packed once to pinned memory in their own pixel format, are cut into contiguous shards of about equal modelled
// cost, and each device copies, converts and scans its own shard.  The result equals RunCascadeDecoded's.
func (pg *Pigo) RunCascadeDecodedSharded(imgs []image.Image, cp CascadeParams, angles []float64) [][]Detection {
	n := len(imgs)
	angles = decodedAngles("RunCascadeDecodedSharded", angles, n)
	if n == 0 {
		return nil
	}
	desc, free := packDecoded(imgs)
	defer free()
	return runCapped(n, func(buf *C.pigo_det, capacity C.int, cnt *C.int) C.int {
		return C.pigo_run_cascade_decoded_sharded(pg.h, &desc[0], C.int(n), anglesPtr(angles), C.int(cp.MinSize), C.int(cp.MaxSize),
			C.double(cp.ShiftFactor), C.double(cp.ScaleFactor), buf, capacity, cnt)
	})
}

// DetectDecoded is DetectImagesAngles on RgbToGrayscale(ImgToNRGBA(img)) of every decoded image: one conversion into device
// memory, then the whole face -> pupils -> landmarks sequence there.  angles is nil (every image at 0) or has one entry per
// image; pp.Angle is not used.  With pp.Sharded the packed images are spread over the GPUs of InitDevices
// (pigo_detect_decoded_sharded): each device copies, converts and runs its own shard, with the same result.
func (pg *Pigo) DetectDecoded(plc *PuplocCascade, calls []LandmarkCall, imgs []image.Image, cp CascadeParams, pp PipelineParams, angles []float64) [][]FaceResult {
	n := len(imgs)
	angles = decodedAngles("DetectDecoded", angles, n)
	if n == 0 {
		return nil
	}
	var images []C.pigo_image
	var desc []C.pigo_decoded
	var free func()
	if pp.Sharded {
		desc, free = packDecoded(imgs) // the host planes, read by the call
	} else {
		images, free = grayDecoded(imgs)
	}
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
				return C.pigo_detect_decoded_sharded(pg.h, plc.h, hs, &fl[0], C.int(ncalls), &desc[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])),
					&prm, nil, C.uint64_t(key), &faces[0], C.int(faceCap), &nfaces[0], &points[0])
			}
			return C.pigo_detect_images_angles(pg.h, plc.h, hs, &fl[0], C.int(ncalls), &images[0], C.int(n), (*C.double)(unsafe.Pointer(&angles[0])),
				&prm, nil, C.uint64_t(key), &faces[0], C.int(faceCap), &nfaces[0], &points[0], C.PIGO_FRAMES_DEVICE, nil)
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
