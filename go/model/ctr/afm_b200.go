// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package model/ctr.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain (see INTEGRATION.md).  Every C call below is
// mirrored one-to-one by the ctypes binding in gorse_b200/_lib.py (gorse_b200.FMRanker), which the GPU test-suite exercises.
//
// Build:  go build -tags "b200 cgo" ./...   with  CGO_CFLAGS=-I<repo>/include  CGO_LDFLAGS="-L<repo>/gorse_b200 -lgorse_b200"
// (*AFM).B200Ranker uploads a trained AFM once; (*AFMB200).Rank ranks the candidates of many users in one call, as
// rankByClickTroughRate (worker/pipeline.go:450-499) does for one user with BatchPredict (fm.go:180-229) and
// cache.SortDocuments.  Inference only: Fit, the XLA AFM and the LLM ranker are unchanged.
//go:build b200 && cgo && !xla

package ctr

/*
#cgo LDFLAGS: -lgorse_b200
#include <stdlib.h>
#include <string.h>
#include "gorse_b200.h"
*/
import "C"

import (
	"errors"
	"sync"
	"unsafe"

	"github.com/gorse-io/gorse/dataset"
)

func afmB200Error(st C.int32_t) error {
	if st == C.GORSE_B200_OK {
		return nil
	}
	return errors.New(C.GoString(C.gorse_b200_last_error()))
}

var (
	afmB200Once sync.Once
	afmB200Ctx  *C.gorse_b200_ctx
	afmB200Err  error
)

func afmB200Context() (*C.gorse_b200_ctx, error) {
	afmB200Once.Do(func() { afmB200Err = afmB200Error(C.gorse_b200_ctx_create(0, &afmB200Ctx)) })
	return afmB200Ctx, afmB200Err
}

// AFMB200 is a trained AFM resident on the GPU.  It holds the model's encoders to build the factored input; it is
// read-only and safe for concurrent Rank calls.  Close releases the device copy.
type AFMB200 struct {
	fm *AFM
	h  *C.gorse_b200_fm
}

// B200Ranker uploads fm.Parameters() (fm.go:136-146) in order: B, V, W, then per slot H, AW, Ab, EW, Eb.
func (fm *AFM) B200Ranker() (*AFMB200, error) {
	ctx, err := afmB200Context()
	if err != nil {
		return nil, err
	}
	fm.mu.RLock()
	defer fm.mu.RUnlock()
	var params []float32
	for _, p := range fm.Parameters() {
		params = append(params, p.Data()...)
	}
	dims := make([]C.int32_t, len(fm.embeddingDim)+1)
	for i, d := range fm.embeddingDim {
		dims[i] = C.int32_t(d)
	}
	r := &AFMB200{fm: fm}
	st := C.gorse_b200_fm_create(ctx, C.int64_t(fm.numFeatures), C.int32_t(fm.nFactors), C.int32_t(fm.numDimension),
		C.int32_t(fm.batchSize), C.int32_t(len(fm.embeddingDim)), (*C.int32_t)(unsafe.Pointer(&dims[0])),
		(*C.float)(unsafe.Pointer(&params[0])), C.int64_t(len(params)), &r.h)
	if err := afmB200Error(st); err != nil {
		return nil, err
	}
	return r, nil
}

// Close frees the device copy of the model.
func (r *AFMB200) Close() {
	if r.h != nil {
		C.gorse_b200_fm_destroy(r.h)
		r.h = nil
	}
}

// features CSR: the id feature (or -1) and the known labels with applyScalers' values (fm.go:232-245), in label order
type afmFeats struct {
	feat []C.int32_t
	off  []C.int64_t
	idx  []C.int32_t
	val  []C.float
}

func (r *AFMB200) appendRow(f *afmFeats, id int32, labels []Label, encodeLabel func(string) int32) {
	if len(f.off) == 0 {
		f.off = append(f.off, 0)
	}
	f.feat = append(f.feat, C.int32_t(id))
	for _, l := range labels {
		if j := encodeLabel(l.Name); j != dataset.NotId {
			v := l.Value
			if r.fm.autoScale {
				if s, ok := r.fm.Scalers[j]; ok {
					v = s.Transform(v)
				}
			}
			f.idx = append(f.idx, C.int32_t(j))
			f.val = append(f.val, C.float(v))
		}
	}
	f.off = append(f.off, C.int64_t(len(f.idx)))
}

func ptrI32(s []C.int32_t) *C.int32_t {
	if len(s) == 0 {
		return nil
	}
	return &s[0]
}

// Rank scores and orders, for each user u, the candidates cands[u] (indices into itemIds).  userLabels / itemLabels and
// itemEmbeddings are what rankByClickTroughRate passes to BatchPredict for the user and for each item.  It returns the scores
// in candidate order and each user's candidate positions by score descending (exact ties by position, NaN last; the
// reference's sort.Slice leaves tie order unpinned).
func (r *AFMB200) Rank(userIds []string, userLabels [][]Label, itemIds []string, itemLabels [][]Label, itemEmbeddings [][]Embedding,
	cands [][]int32) (scores [][]float32, order [][]int32, err error) {
	if len(userIds) == 0 {
		return nil, nil, nil
	}
	fm := r.fm
	fm.mu.RLock()
	defer fm.mu.RUnlock()
	var users, items afmFeats
	for u, id := range userIds {
		r.appendRow(&users, fm.Index.EncodeUser(id), userLabels[u], fm.Index.EncodeUserLabel)
	}
	for i, id := range itemIds {
		r.appendRow(&items, fm.Index.EncodeItem(id), itemLabels[i], fm.Index.EncodeItemLabel)
	}
	// embeddings per slot in C memory (an array of pointers into Go memory may not cross into C), with the presence mask
	// of BatchPredict's rule: a known name and the slot's length (fm.go:208-227)
	nEmb := len(fm.embeddingDim)
	mask := make([]C.uint8_t, len(itemIds)*nEmb+1)
	slots := (*[1 << 20]*C.uint16_t)(C.malloc(C.size_t(nEmb+1) * C.size_t(unsafe.Sizeof(uintptr(0)))))
	defer C.free(unsafe.Pointer(slots))
	for s := 0; s < nEmb; s++ {
		bytes := C.size_t(len(itemIds)*fm.embeddingDim[s]*2 + 2)
		slots[s] = (*C.uint16_t)(C.malloc(bytes))
		defer C.free(unsafe.Pointer(slots[s]))
		C.memset(unsafe.Pointer(slots[s]), 0, bytes)
	}
	if fm.embeddingIndex != nil {
		for i := range itemIds {
			for _, e := range itemEmbeddings[i] {
				s := fm.embeddingIndex.ToNumber(e.Name)
				if s == dataset.NotId || len(e.Value) != fm.embeddingDim[s] || len(e.Value) == 0 {
					continue
				}
				mask[i*nEmb+int(s)] = 1
				dst := unsafe.Add(unsafe.Pointer(slots[s]), i*fm.embeddingDim[s]*2)
				C.memcpy(dst, unsafe.Pointer(&e.Value[0]), C.size_t(len(e.Value)*2))
			}
		}
	}
	candOff := make([]C.int64_t, 1, len(userIds)+1)
	var candItems []C.int32_t
	for _, c := range cands {
		for _, i := range c {
			candItems = append(candItems, C.int32_t(i))
		}
		candOff = append(candOff, C.int64_t(len(candItems)))
	}
	flatScores := make([]float32, len(candItems)+1)
	flatOrder := make([]int32, len(candItems)+1)
	users.idx, users.val = append(users.idx, 0), append(users.val, 0)
	items.idx, items.val = append(items.idx, 0), append(items.val, 0)
	if len(items.off) == 0 {
		items.off = []C.int64_t{0}
	}
	st := C.gorse_b200_fm_rank(r.h, C.int64_t(len(userIds)), ptrI32(users.feat), &users.off[0], &users.idx[0], &users.val[0],
		C.int64_t(len(itemIds)), ptrI32(items.feat), &items.off[0], &items.idx[0], &items.val[0],
		(**C.uint16_t)(unsafe.Pointer(slots)), &mask[0], &candOff[0], ptrI32(candItems),
		(*C.float)(unsafe.Pointer(&flatScores[0])), (*C.int32_t)(unsafe.Pointer(&flatOrder[0])), nil)
	if err = afmB200Error(st); err != nil {
		return nil, nil, err
	}
	scores, order = make([][]float32, len(cands)), make([][]int32, len(cands))
	for u := range cands {
		a, b := candOff[u], candOff[u+1]
		scores[u], order[u] = flatScores[a:b], flatOrder[a:b]
	}
	return scores, order, nil
}
