// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package main of cmd/gorse-bench.
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image).  The C call below is mirrored one-to-one by the
// ctypes binding in gorse_b200/_lib.py (gorse_b200.evaluate_embeddings), which the GPU test-suite exercises.
//
// scoreEmbeddings on the GPU: `gorse-bench embedding`'s per-user scoring (EvaluateEmbedding, main.go:403-465) in one
// gorse_b200_embedding_eval call.  The extraction of the embeddings, including the OpenAI text path, stays in
// EvaluateEmbedding; INTEGRATION.md ("gorse-bench embedding") shows the edit that calls this function and moves the
// reference's loop, unchanged, into scoreEmbeddingsCPU.  Built without the tags, embedding_cpu.go makes that loop
// scoreEmbeddings.
//go:build b200 && cgo

package main

/*
#include "gorse_b200.h"
*/
import "C"

import (
	"sync"

	"github.com/gorse-io/gorse/common/log"
	"github.com/gorse-io/gorse/dataset"
	"github.com/gorse-io/gorse/model/cf"
	"go.uber.org/zap"
)

var (
	embeddingCtxOnce sync.Once
	embeddingCtx     *C.gorse_b200_ctx
	embeddingCtxSt   C.int32_t
)

func embeddingCSR(rows [][]int32) ([]int64, []int32) {
	off := make([]int64, len(rows)+1)
	for i, r := range rows {
		off[i+1] = off[i] + int64(len(r))
	}
	items := make([]int32, 0, off[len(rows)]+1)
	for _, r := range rows {
		items = append(items, r...)
	}
	return off, append(items, 0) // never empty, so &items[0] is valid
}

// scoreEmbeddings flattens the embeddings into one row-major table with a presence mask, passes the shots (train), the
// test items and the negatives as CSRs, and makes one call.  The negatives are the ones SampleUserNegatives cached for the
// dataset when main called it (dataset.go:242-253), the same the CPU path ranks, so both paths score the same candidates.
// Embeddings of different lengths (the text path does not check them, main.go:346-380) and library errors are logged,
// and the reference's loop scores instead.
func scoreEmbeddings(train, test dataset.CFSplit, embeddings [][]float32, topK, jobs int) cf.Score {
	dim := 0
	for _, e := range embeddings {
		if e != nil {
			dim = len(e)
			break
		}
	}
	if dim == 0 || test.CountUsers() == 0 {
		return scoreEmbeddingsCPU(train, test, embeddings, topK, jobs)
	}
	for i, e := range embeddings {
		if e != nil && len(e) != dim {
			log.Logger().Error("embeddings of different lengths; scoring on the CPU",
				zap.Int("item", i), zap.Int("expected", dim), zap.Int("got", len(e)))
			return scoreEmbeddingsCPU(train, test, embeddings, topK, jobs)
		}
	}
	flat := make([]float32, len(embeddings)*dim)
	mask := make([]uint8, len(embeddings)+1)
	for i, e := range embeddings {
		if e != nil {
			copy(flat[i*dim:(i+1)*dim], e)
			mask[i] = 1
		}
	}
	shotOff, shotItems := embeddingCSR(train.GetUserFeedback())
	testOff, testItems := embeddingCSR(test.GetUserFeedback())
	negOff, negItems := embeddingCSR(test.SampleUserNegatives(train, 99))

	embeddingCtxOnce.Do(func() { embeddingCtxSt = C.gorse_b200_ctx_create(0, &embeddingCtx) })
	st := embeddingCtxSt
	var out [3]C.float
	var users C.int64_t
	if st == C.GORSE_B200_OK {
		st = C.gorse_b200_embedding_eval(embeddingCtx, C.int32_t(len(embeddings)), C.int32_t(dim), (*C.float)(&flat[0]),
			(*C.uint8_t)(&mask[0]), C.int64_t(test.CountUsers()), (*C.int64_t)(&shotOff[0]), (*C.int32_t)(&shotItems[0]),
			(*C.int64_t)(&testOff[0]), (*C.int32_t)(&testItems[0]), nil, nil, (*C.int64_t)(&negOff[0]), (*C.int32_t)(&negItems[0]),
			99, 0, C.int32_t(topK), &out[0], &users)
	}
	if st != C.GORSE_B200_OK {
		log.Logger().Error("gorse_b200_embedding_eval failed; scoring on the CPU",
			zap.Int32("status", int32(st)), zap.String("error", C.GoString(C.gorse_b200_last_error())))
		return scoreEmbeddingsCPU(train, test, embeddings, topK, jobs)
	}
	return cf.Score{NDCG: float32(out[0]), Precision: float32(out[1]), Recall: float32(out[2])}
}
