// refdump -- runs the UNMODIFIED Go reference (github.com/esimov/pigo/core) on raw grayscale buffers and dumps what it
// returns, so that the CPU oracle (oracle/pigo_oracle.c) can be pinned to true reference outputs on any box that has a Go
// toolchain (see DESIGN.md section 2).
//
// Build / run (offline, against the vendored module; nothing is written into the reference tree):
//
//	python tools/refdump/make_inputs.py                      # writes oracle/_ref/inputs/{manifest.json,*.u8}
//	cd $PIGO_REF && GOFLAGS=-mod=vendor \
//	    go run $REPO/tools/refdump/main.go -in $REPO/oracle/_ref/inputs -out $REPO/oracle/_ref/refdump.json
//	python -m pytest tests/test_refdump.py                   # consumes the dump (skips while it is absent)
//
// What is dumped, per input buffer and parameter set of the manifest:
//   - (*Pigo).RunCascade(cp, angle)            core/pigo.go:212-258   every detection: Row, Col, Scale and math.Float32bits(Q)
//   - (*Pigo).ClusterDetections(dets, iou)     core/pigo.go:262-308   the in-place sorted input AND the clusters
//   - (*PuplocCascade).RunDetector             core/puploc.go:239-277 with the global math/rand stream made reproducible by
//     rand.Seed(s): the same stream is replayed from rand.New(rand.NewSource(s)) and dumped as the `randoms` the oracle and
//     the CUDA library take as an injected argument (3 float32 per perturbation, row/col/scale order).  The first call in
//     the process uses Perturbs < 63 on a FRESH sync.Pool object (zeros in the unused slots), every later call uses
//     Perturbs = 63, so stale pool contents never matter (SURVEY.md Q10).
//   - (*PuplocCascade).GetLandmarkPoint        core/flploc.go:36-57   same seeding scheme
package main

import (
	"encoding/json"
	"flag"
	"log"
	"math"
	"math/rand"
	"os"
	"path/filepath"

	pigo "github.com/esimov/pigo/core"
)

type input struct {
	File string `json:"file"`
	Rows int    `json:"rows"`
	Cols int    `json:"cols"`
	Dim  int    `json:"dim"`
	Runs []struct {
		MinSize     int       `json:"min_size"`
		MaxSize     int       `json:"max_size"`
		ShiftFactor float64   `json:"shift_factor"`
		ScaleFactor float64   `json:"scale_factor"`
		Angle       float64   `json:"angle"`
		IoU         []float64 `json:"iou"`
	} `json:"runs"`
	Pupils []struct {
		Cascade  string  `json:"cascade"` // file name under the cascade directory, e.g. "puploc" or "lps/lp42"
		Row      int     `json:"row"`
		Col      int     `json:"col"`
		Scale    float32 `json:"scale"`
		Perturbs int     `json:"perturbs"`
		Angle    float64 `json:"angle"`
		FlipV    bool    `json:"flipv"`
		Seed     int64   `json:"seed"`
	} `json:"pupils"`
	Landmarks []struct {
		Cascade  string `json:"cascade"`
		LeftRow  int    `json:"left_row"`
		LeftCol  int    `json:"left_col"`
		RightRow int    `json:"right_row"`
		RightCol int    `json:"right_col"`
		Perturbs int    `json:"perturbs"`
		FlipV    bool   `json:"flipv"`
		Seed     int64  `json:"seed"`
	} `json:"landmarks"`
}

type det struct {
	Row   int    `json:"row"`
	Col   int    `json:"col"`
	Scale int    `json:"scale"`
	QBits uint32 `json:"q_bits"`
}

func toDets(d []pigo.Detection) []det {
	out := make([]det, len(d))
	for i, x := range d {
		out[i] = det{x.Row, x.Col, x.Scale, math.Float32bits(x.Q)}
	}
	return out
}

func drawn(seed int64, n int) []uint32 {
	r := rand.New(rand.NewSource(seed))
	out := make([]uint32, n)
	for i := range out {
		out[i] = math.Float32bits(r.Float32())
	}
	return out
}

func main() {
	in := flag.String("in", "oracle/_ref/inputs", "directory with manifest.json and the raw buffers")
	out := flag.String("out", "oracle/_ref/refdump.json", "output file")
	casc := flag.String("cascade", "cascade", "cascade directory of the reference (run from the reference checkout)")
	flag.Parse()

	mf, err := os.ReadFile(filepath.Join(*in, "manifest.json"))
	if err != nil {
		log.Fatal(err)
	}
	var inputs []input
	if err := json.Unmarshal(mf, &inputs); err != nil {
		log.Fatal(err)
	}
	ff, err := os.ReadFile(filepath.Join(*casc, "facefinder"))
	if err != nil {
		log.Fatal(err)
	}
	classifier, err := pigo.NewPigo().Unpack(ff)
	if err != nil {
		log.Fatal(err)
	}
	plcs := map[string]*pigo.PuplocCascade{}
	getPlc := func(name string) *pigo.PuplocCascade {
		if p, ok := plcs[name]; ok {
			return p
		}
		b, err := os.ReadFile(filepath.Join(*casc, name))
		if err != nil {
			log.Fatal(err)
		}
		p, err := pigo.NewPuplocCascade().UnpackCascade(b)
		if err != nil {
			log.Fatal(err)
		}
		plcs[name] = p
		return p
	}

	type runOut struct {
		Params   interface{}      `json:"params"`
		Dets     []det            `json:"detections"`
		Sorted   map[string][]det `json:"sorted_by_iou"`
		Clusters map[string][]det `json:"clusters_by_iou"`
	}
	type pupOut struct {
		Params  interface{} `json:"params"`
		Randoms []uint32    `json:"randoms_bits"`
		Row     int         `json:"row"`
		Col     int         `json:"col"`
		Scale   uint32      `json:"scale_bits"`
	}
	type fileOut struct {
		File      string   `json:"file"`
		Runs      []runOut `json:"runs"`
		Pupils    []pupOut `json:"pupils"`
		Landmarks []pupOut `json:"landmarks"`
	}
	var result struct {
		GoVersion string    `json:"go_version"`
		Files     []fileOut `json:"files"`
	}
	result.GoVersion = goVersion()
	for _, inp := range inputs {
		px, err := os.ReadFile(filepath.Join(*in, inp.File))
		if err != nil {
			log.Fatal(err)
		}
		img := pigo.ImageParams{Pixels: px, Rows: inp.Rows, Cols: inp.Cols, Dim: inp.Dim}
		fo := fileOut{File: inp.File}
		for _, r := range inp.Runs {
			cp := pigo.CascadeParams{MinSize: r.MinSize, MaxSize: r.MaxSize, ShiftFactor: r.ShiftFactor, ScaleFactor: r.ScaleFactor, ImageParams: img}
			dets := classifier.RunCascade(cp, r.Angle)
			ro := runOut{Params: r, Dets: toDets(dets), Sorted: map[string][]det{}, Clusters: map[string][]det{}}
			for _, iou := range r.IoU {
				cpy := append([]pigo.Detection(nil), dets...)
				cl := classifier.ClusterDetections(cpy, iou)
				key := jsonKey(iou)
				ro.Sorted[key] = toDets(cpy) // ClusterDetections sorts its argument in place (core/pigo.go:264)
				ro.Clusters[key] = toDets(cl)
			}
			fo.Runs = append(fo.Runs, ro)
		}
		for _, p := range inp.Pupils {
			rand.Seed(p.Seed) //nolint:staticcheck // deliberate: makes the reference's global stream reproducible
			res := getPlc(p.Cascade).RunDetector(pigo.Puploc{Row: p.Row, Col: p.Col, Scale: p.Scale, Perturbs: p.Perturbs}, img, p.Angle, p.FlipV)
			fo.Pupils = append(fo.Pupils, pupOut{Params: p, Randoms: drawn(p.Seed, 3*p.Perturbs), Row: res.Row, Col: res.Col, Scale: math.Float32bits(res.Scale)})
		}
		for _, l := range inp.Landmarks {
			rand.Seed(l.Seed) //nolint:staticcheck
			le := &pigo.Puploc{Row: l.LeftRow, Col: l.LeftCol}
			re := &pigo.Puploc{Row: l.RightRow, Col: l.RightCol}
			res := getPlc(l.Cascade).GetLandmarkPoint(le, re, img, l.Perturbs, l.FlipV)
			fo.Landmarks = append(fo.Landmarks, pupOut{Params: l, Randoms: drawn(l.Seed, 3*l.Perturbs), Row: res.Row, Col: res.Col, Scale: math.Float32bits(res.Scale)})
		}
		result.Files = append(result.Files, fo)
	}
	b, err := json.MarshalIndent(result, "", " ")
	if err != nil {
		log.Fatal(err)
	}
	if err := os.WriteFile(*out, b, 0o644); err != nil {
		log.Fatal(err)
	}
	log.Printf("wrote %s (%d inputs)", *out, len(result.Files))
}

func jsonKey(f float64) string {
	b, _ := json.Marshal(f)
	return string(b)
}
