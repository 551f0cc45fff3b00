// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package model/ctr.
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image).  The C call below is mirrored one-to-one by the
// ctypes binding in gorse_b200/_lib.py (gorse_b200.ranker_gauc), which the GPU test-suite exercises.
//
// (*AFM).GAUCB200 is the scoring of `gorse-bench reranker`'s AFM half after the fit (EvaluateAFM,
// cmd/gorse-bench/main.go:133-206) in one gorse_b200_fm_gauc call: BatchInternalPredict on the whole test split in test
// order, then the per-user AUC and GAUC.  cmd/gorse-bench/reranker_b200.go calls it.
//go:build b200 && cgo && !xla

package ctr

/*
#include "gorse_b200.h"
*/
import "C"

import (
	"unsafe"

	"github.com/gorse-io/gorse/dataset"
)

// UserAUC is one scored user of GAUCB200: its index, its positive training rows, its test rows and its AUC.
type UserAUC struct {
	User       int32
	Feedback   int
	Candidates int
	AUC        float32
}

// GAUCB200 scores the fitted model on testSet.  feedbackCount[u] is the number of training rows with target > 0 whose
// first index is u (main.go:133-140), for every user index the test rows hold; contextSize is cfg.Recommend.ContextSize.
// The users come back in ascending index order (the reference visits them in map order).
func (fm *AFM) GAUCB200(testSet dataset.CTRSplit, feedbackCount []int64, contextSize int) (float64, []UserAUC, error) {
	c, err := afmB200Context()
	if err != nil {
		return 0, nil, err
	}
	var params []float32
	for _, p := range fm.Parameters() {
		params = append(params, p.Data()...)
	}
	off, idx, val, tgt := fm.b200Rows(testSet, fm.autoScale) // BatchInternalPredict scales when autoScale is set
	nEmb := len(fm.embeddingDim)
	table, rows := b200EmbTable(fm.embeddingDim, testSet)
	defer table.free()
	dims := append(append([]C.int32_t{}, table.dims...), 0)
	nUsers := len(feedbackCount)
	fb := append(append([]int64{}, feedbackCount...), 0)
	users := make([]C.int32_t, nUsers+1)
	feedback := make([]C.int64_t, nUsers+1)
	cand := make([]C.int64_t, nUsers+1)
	auc := make([]C.float, nUsers+1)
	var nScored C.int64_t
	var gauc C.double
	var slots **C.uint16_t
	if nEmb > 0 {
		slots = (**C.uint16_t)(unsafe.Pointer(table.slots))
	}
	// the library copies during the call and keeps no Go pointer (cgo rule)
	st := C.gorse_b200_fm_gauc(c, C.int64_t(fm.numFeatures), C.int32_t(fm.nFactors), C.int32_t(fm.numDimension),
		C.int32_t(fm.batchSize), C.int32_t(nEmb), &dims[0], (*C.float)(unsafe.Pointer(&params[0])), C.int64_t(len(params)),
		C.int64_t(testSet.Count()), &off[0], ptrI32(idx), ptrF32(val), ptrF32(tgt), &rows[0][0], C.int64_t(table.rows), slots,
		&table.mask[0], C.int64_t(nUsers), (*C.int64_t)(unsafe.Pointer(&fb[0])), C.int64_t(contextSize), nil, &users[0],
		&feedback[0], &cand[0], &auc[0], &nScored, &gauc, nil)
	if err := afmB200Error(st); err != nil {
		return 0, nil, err
	}
	out := make([]UserAUC, nScored)
	for j := range out {
		out[j] = UserAUC{User: int32(users[j]), Feedback: int(feedback[j]), Candidates: int(cand[j]), AUC: float32(auc[j])}
	}
	return float64(gauc), out, nil
}
