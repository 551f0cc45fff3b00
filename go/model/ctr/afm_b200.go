// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package model/ctr.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain (see INTEGRATION.md).  Every C call below is
// mirrored one-to-one by the ctypes binding in gorse_b200/_lib.py (gorse_b200.FMRanker), which the GPU test-suite exercises.
//
// Build:  go build -tags "b200 cgo" ./...   with  CGO_CFLAGS=-I<repo>/include  CGO_LDFLAGS="-L<repo>/gorse_b200 -lgorse_b200"
// (*AFM).B200Ranker uploads a trained AFM once; (*AFMB200).Rank ranks the candidates of many users in one call, as
// rankByClickTroughRate (worker/pipeline.go:450-499) does for one user with BatchPredict (fm.go:180-229) and
// cache.SortDocuments.  (*AFM).Fit trains on the GPU: a model without embedding slots through gorse_b200_fm_fit, one with
// slots through gorse_b200_fm_fit_emb; a model beyond the library's limits trains with the reference's Fit, which the
// integration renames fitCPU (INTEGRATION.md; fm_fit_cpu.go keeps the name Fit for builds without the tag).  The XLA AFM
// and the LLM ranker are unchanged.
//go:build b200 && cgo && !xla

package ctr

/*
#cgo LDFLAGS: -lgorse_b200
#include <stdlib.h>
#include <string.h>
#include "gorse_b200.h"

// cgo cannot call Go closures from C directly: Fit's progress callback goes through this exported trampoline.
extern int32_t gorseB200FMProgress(void *user, int32_t epoch, int32_t nEpochs, float auc);
static int32_t gorse_b200_fm_progress_tramp(void *user, int32_t epoch, int32_t n, float auc) {
    return gorseB200FMProgress(user, epoch, n, auc);
}
static gorse_b200_progress_fn gorse_b200_fm_progress_ptr(void) { return gorse_b200_fm_progress_tramp; }
*/
import "C"

import (
	"context"
	"errors"
	"fmt"
	"runtime/cgo"
	"sync"
	"unsafe"

	"github.com/gorse-io/gorse/common/log"
	"github.com/gorse-io/gorse/common/monitor"
	"github.com/gorse-io/gorse/dataset"
	"github.com/gorse-io/gorse/model"
	"go.uber.org/zap"
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

// ---- training ------------------------------------------------------------------------------------------------------

// the CTR rows of a split in dataset order as a CSR; scale applies fm.Scalers to the values: Fit does so for the
// training rows (fm.go:331-344), and BatchInternalPredict for the test rows when autoScale is set (fm.go:159-165)
func (fm *AFM) b200Rows(set dataset.CTRSplit, scale bool) (off []C.int64_t, idx []C.int32_t, val []C.float, tgt []C.float) {
	off = make([]C.int64_t, 1, set.Count()+1)
	tgt = make([]C.float, 0, set.Count()+1)
	for i := 0; i < set.Count(); i++ {
		indices, values, _, target := set.Get(i)
		for j, x := range indices {
			v := values[j]
			if scale {
				if s, ok := fm.Scalers[x]; ok {
					v = s.Transform(v)
				}
			}
			idx = append(idx, C.int32_t(x))
			val = append(val, C.float(v))
		}
		off = append(off, C.int64_t(len(idx)))
		tgt = append(tgt, C.float(target))
	}
	return off, idx, val, tgt
}

// afmEmbTable is the item-embedding table of a fit in C memory (an array of pointers into Go memory may not cross into C):
// one row per distinct item of the splits, bf16 bits per slot, and the presence mask of convertToTensors' rule
// (fm.go:555-561): the slot exists for the item and has the slot's length.
type afmEmbTable struct {
	dims  []C.int32_t
	slots *[1 << 20]*C.uint16_t
	mask  []C.uint8_t
	rows  int
}

func (t *afmEmbTable) free() {
	for s := range t.dims {
		C.free(unsafe.Pointer(t.slots[s]))
	}
	C.free(unsafe.Pointer(t.slots))
}

// b200EmbTable builds the table and the table row of every sample of the splits (-1: the sample has no embeddings).
// CTRSplit.Get hands out ItemEmbeddings[Items[i]] (model/ctr/data.go:221-240), so samples of one item share one slice:
// its identity is the item, and the splits of one dataset share the item table.
func b200EmbTable(dims []int, sets ...dataset.CTRSplit) (*afmEmbTable, [][]C.int32_t) {
	rowOf := make(map[*[]uint16]int32)
	var items [][][]uint16
	sampleRows := make([][]C.int32_t, len(sets))
	for q, set := range sets {
		sampleRows[q] = make([]C.int32_t, set.Count()+1)
		for i := 0; i < set.Count(); i++ {
			_, _, e, _ := set.Get(i)
			if len(e) == 0 {
				sampleRows[q][i] = -1
				continue
			}
			r, ok := rowOf[&e[0]]
			if !ok {
				r = int32(len(items))
				rowOf[&e[0]] = r
				items = append(items, e)
			}
			sampleRows[q][i] = C.int32_t(r)
		}
	}
	nEmb := len(dims)
	t := &afmEmbTable{dims: make([]C.int32_t, nEmb), mask: make([]C.uint8_t, len(items)*nEmb+1), rows: len(items)}
	t.slots = (*[1 << 20]*C.uint16_t)(C.malloc(C.size_t(nEmb+1) * C.size_t(unsafe.Sizeof(uintptr(0)))))
	for s, d := range dims {
		t.dims[s] = C.int32_t(d)
		bytes := C.size_t(len(items)*d*2 + 2)
		t.slots[s] = (*C.uint16_t)(C.malloc(bytes))
		C.memset(unsafe.Pointer(t.slots[s]), 0, bytes)
		for r, e := range items {
			if len(e) > s && len(e[s]) == d && d > 0 {
				t.mask[r*nEmb+s] = 1
				C.memcpy(unsafe.Add(unsafe.Pointer(t.slots[s]), r*d*2), unsafe.Pointer(&e[s][0]), C.size_t(d*2))
			}
		}
	}
	return t, sampleRows
}

func ptrF32(s []C.float) *C.float {
	if len(s) == 0 {
		return nil
	}
	return &s[0]
}

type afmFitProgress struct {
	ctx     context.Context
	span    *monitor.Span
	nEpochs int
}

//export gorseB200FMProgress
func gorseB200FMProgress(user unsafe.Pointer, epoch, nEpochs C.int32_t, auc C.float) C.int32_t {
	p := (*(*cgo.Handle)(user)).Value().(*afmFitProgress) // user = &handle, the documented way to carry a Handle in a void*
	if epoch > 0 {
		p.span.Add(1) // fm.go:414
	}
	if auc >= 0 {
		log.Logger().Info(fmt.Sprintf("fit AFM %v/%v", int(epoch), p.nEpochs), zap.Float32("AUC", float32(auc)))
	}
	if p.ctx.Err() != nil {
		return 1 // Fit returns Score{} where the reference checks ctx.Err(), before the next batch (fm.go:364-367)
	}
	return 0
}

// Fit is AFM.Fit (fm.go:307-417) on the GPU, step for step as the reference: Init stays here, the library gets
// fm.Parameters() and the scaled rows, and the fitted parameters are copied back into the model's tensors.  A model with
// item-embedding slots also sends the splits' item-embedding table and every sample's row of it (gorse_b200_fm_fit_emb).
// Only GORSE_B200_ERR_UNSUPPORTED from the library (more than 32 factors, 8 slots or an embedding wider than 1024) trains
// with the reference's Fit (fitCPU).
func (fm *AFM) Fit(ctx context.Context, trainSet, testSet dataset.CTRSplit, config *FitConfig) Score {
	c, err := afmB200Context()
	if err != nil {
		log.Logger().Error("gorse_b200 context", zap.Error(err))
		return Score{}
	}
	log.Logger().Info("fit AFM on the GPU",
		zap.Int("train_set_size", trainSet.Count()),
		zap.Int("test_set_size", testSet.Count()),
		zap.Any("params", fm.GetParams()),
		zap.Any("config", config))
	fm.Init(trainSet)
	var params []float32
	for _, p := range fm.Parameters() {
		params = append(params, p.Data()...)
	}
	trOff, trIdx, trVal, trTgt := fm.b200Rows(trainSet, true)
	teOff, teIdx, teVal, teTgt := fm.b200Rows(testSet, fm.autoScale)
	var p C.gorse_b200_fm_fit_params
	p.n_factors, p.n_epochs, p.lr, p.reg = C.int32_t(fm.nFactors), C.int32_t(fm.nEpochs), C.float(fm.lr), C.float(fm.reg)
	switch fm.optimizer {
	case model.SGD:
		p.optimizer = C.GORSE_B200_FM_SGD
	case model.Adam:
		p.optimizer = C.GORSE_B200_FM_ADAM
	default:
		panic("unknown optimizer")
	}
	p.batch_size, p.verbose, p.patience = C.int32_t(fm.batchSize), C.int32_t(config.Verbose), C.int32_t(config.Patience)

	_, span := monitor.Start(ctx, "FM.Fit", fm.nEpochs)
	defer span.End()
	h := cgo.NewHandle(&afmFitProgress{ctx: ctx, span: span, nEpochs: fm.nEpochs})
	defer h.Delete()
	out := make([]float32, len(params))
	var res C.gorse_b200_fm_fit_result
	// the library copies during the call and keeps no Go pointer (cgo rule)
	var st C.int32_t
	if len(fm.embeddingDim) == 0 {
		st = C.gorse_b200_fm_fit(c, C.int64_t(fm.numFeatures), C.int32_t(fm.numDimension), 0, &p,
			C.int64_t(trainSet.Count()), &trOff[0], ptrI32(trIdx), ptrF32(trVal), ptrF32(trTgt),
			C.int64_t(testSet.Count()), &teOff[0], ptrI32(teIdx), ptrF32(teVal), ptrF32(teTgt),
			(*C.float)(unsafe.Pointer(&params[0])), C.int64_t(len(params)), (*C.float)(unsafe.Pointer(&out[0])), nil,
			C.gorse_b200_fm_progress_ptr(), unsafe.Pointer(&h), &res)
	} else {
		table, rows := b200EmbTable(fm.embeddingDim, trainSet, testSet)
		defer table.free()
		st = C.gorse_b200_fm_fit_emb(c, C.int64_t(fm.numFeatures), C.int32_t(fm.numDimension), &p,
			C.int64_t(trainSet.Count()), &trOff[0], ptrI32(trIdx), ptrF32(trVal), ptrF32(trTgt), &rows[0][0],
			C.int64_t(testSet.Count()), &teOff[0], ptrI32(teIdx), ptrF32(teVal), ptrF32(teTgt), &rows[1][0],
			C.int32_t(len(table.dims)), &table.dims[0], C.int64_t(table.rows), (**C.uint16_t)(unsafe.Pointer(table.slots)), &table.mask[0],
			(*C.float)(unsafe.Pointer(&params[0])), C.int64_t(len(params)), (*C.float)(unsafe.Pointer(&out[0])), nil,
			C.gorse_b200_fm_progress_ptr(), unsafe.Pointer(&h), &res)
	}
	if st == C.GORSE_B200_ERR_UNSUPPORTED {
		log.Logger().Info("gorse_b200 cannot fit this AFM; fitting on the CPU", zap.Error(afmB200Error(st)))
		return fm.fitCPU(ctx, trainSet, testSet, config)
	}
	if err := afmB200Error(st); err != nil {
		log.Logger().Error("gorse_b200 fm_fit", zap.Error(err))
		return Score{}
	}
	o := 0
	for _, t := range fm.Parameters() { // B, V, W, then every slot's H, AW, Ab, EW, Eb: the layout params_in had
		o += copy(t.Data(), out[o:])
	}
	if res.cancelled != 0 {
		log.Logger().Info("fit AFM canceled", zap.Error(ctx.Err()))
		return Score{}
	}
	if res.diverged != 0 {
		log.Logger().Warn("model diverged", zap.Float32("lr", fm.lr))
	}
	if res.early_stopped != 0 {
		log.Logger().Info("early stopping", zap.Int("best_epoch", int(res.best_epoch)), zap.Int("patience", config.Patience))
	}
	return Score{Precision: float32(res.precision), Recall: float32(res.recall), Accuracy: float32(res.accuracy), AUC: float32(res.auc)}
}
