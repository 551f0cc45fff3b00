// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package model/ctr.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain (see INTEGRATION.md).  Every C call below is
// mirrored one-to-one by the ctypes binding in gorse_b200/_lib.py (gorse_b200.FMTrainer.fit_trials), which the GPU
// test-suite exercises.
//
// FitTrialsB200 fits the trials of optimizeClickThroughRatePrediction (master/tasks.go:1318-1363) in one
// gorse_b200_fm_fit_trials call; INTEGRATION.md ("The FM model search") shows where the master calls it.
//go:build b200 && cgo && !xla

package ctr

/*
#include <stdlib.h>
#include "gorse_b200.h"

// the per-epoch callback of gorse_b200_fm_fit_trials goes through this exported trampoline (see afm_b200.go)
extern int32_t gorseB200FMTrialsProgress(void *user, int32_t epoch, int32_t nTrials, gorse_b200_fm_trial_state *states);
static int32_t gorse_b200_fm_trials_progress_tramp(void *user, int32_t epoch, int32_t n, const gorse_b200_fm_trial_state *states) {
    return gorseB200FMTrialsProgress(user, epoch, n, (gorse_b200_fm_trial_state *)states);
}
static gorse_b200_fm_trials_progress_fn gorse_b200_fm_trials_progress_ptr(void) { return gorse_b200_fm_trials_progress_tramp; }
*/
import "C"

import (
	"context"
	"errors"
	"runtime/cgo"
	"unsafe"

	"github.com/gorse-io/gorse/common/log"
	"github.com/gorse-io/gorse/common/monitor"
	"github.com/gorse-io/gorse/dataset"
	"github.com/gorse-io/gorse/model"
	"go.uber.org/zap"
)

type fmTrialsProgress struct {
	ctx   context.Context
	spans []*monitor.Span
	run   []int32
}

//export gorseB200FMTrialsProgress
func gorseB200FMTrialsProgress(user unsafe.Pointer, epoch, nTrials C.int32_t, states *C.gorse_b200_fm_trial_state) C.int32_t {
	p := (*(*cgo.Handle)(user)).Value().(*fmTrialsProgress)
	for k := 0; k < int(nTrials); k++ {
		s := (*C.gorse_b200_fm_trial_state)(unsafe.Add(unsafe.Pointer(states), uintptr(k)*unsafe.Sizeof(*states)))
		for ; p.run[k] < int32(s.epochs_run); p.run[k]++ {
			p.spans[k].Add(1) // fm.go:414, once per epoch of each trial
		}
	}
	if p.ctx.Err() != nil {
		return 1 // unfinished trials return Score{} (fm.go:364-367)
	}
	return 0
}

// FitTrialsB200 returns the scores of the trials in trial order: trial k's score is what NewAFM(trials[k]).Fit(ctx,
// trainSet, testSet, config) returns, which is what ModelSearch.Objective compares.  Each trial runs NewAFM and Init here,
// so its parameters start where its solo Fit would start; the rows are built once (the scalers depend on trainSet only).
// The models are discarded, as the reference discards the search's models.  GORSE_B200_ERR_UNSUPPORTED (more than 32
// factors, 8 slots or an embedding wider than 1024), or trials that disagree on autoScale, fit each trial with (*AFM).Fit.
// An error means no trial was fitted.
func FitTrialsB200(ctx context.Context, trials []model.Params, trainSet, testSet dataset.CTRSplit, config *FitConfig) ([]Score, error) {
	if len(trials) == 0 {
		return nil, nil
	}
	c, err := afmB200Context()
	if err != nil {
		return nil, err
	}
	models := make([]*AFM, len(trials))
	for k, t := range trials {
		models[k] = NewAFM(t)
		models[k].Init(trainSet)
	}
	m0 := models[0]
	for _, m := range models {
		if m.autoScale != m0.autoScale {
			log.Logger().Info("AFM trials disagree on autoScale; fitting them one by one")
			return fitTrialsOneByOne(ctx, trials, trainSet, testSet, config), nil
		}
	}
	params := make([]C.gorse_b200_fm_fit_params, len(trials))
	var nParams int
	for _, t := range m0.Parameters() {
		nParams += len(t.Data())
	}
	// params_in / params_out live in C memory: a C array may not hold pointers into Go memory
	bytes := C.size_t(nParams+1) * C.size_t(unsafe.Sizeof(C.float(0)))
	ptrBytes := C.size_t(len(trials)) * C.size_t(unsafe.Sizeof(uintptr(0)))
	pin := (*[1 << 20]*C.float)(C.malloc(ptrBytes))
	pout := (*[1 << 20]*C.float)(C.malloc(ptrBytes))
	defer C.free(unsafe.Pointer(pin))
	defer C.free(unsafe.Pointer(pout))
	for k, m := range models {
		p := &params[k]
		p.n_factors, p.n_epochs, p.lr, p.reg = C.int32_t(m.nFactors), C.int32_t(m.nEpochs), C.float(m.lr), C.float(m.reg)
		switch m.optimizer {
		case model.SGD:
			p.optimizer = C.GORSE_B200_FM_SGD
		case model.Adam:
			p.optimizer = C.GORSE_B200_FM_ADAM
		default:
			panic("unknown optimizer")
		}
		p.batch_size, p.verbose, p.patience = C.int32_t(m.batchSize), C.int32_t(config.Verbose), C.int32_t(config.Patience)
		pin[k] = (*C.float)(C.malloc(bytes))
		pout[k] = (*C.float)(C.malloc(bytes))
		defer C.free(unsafe.Pointer(pin[k]))
		defer C.free(unsafe.Pointer(pout[k]))
		o := 0
		for _, t := range m.Parameters() {
			for _, v := range t.Data() {
				*(*C.float)(unsafe.Add(unsafe.Pointer(pin[k]), o*4)) = C.float(v)
				o++
			}
		}
		if o != nParams {
			return nil, errors.New("AFM trials of different model sizes")
		}
	}
	trOff, trIdx, trVal, trTgt := m0.b200Rows(trainSet, true)
	teOff, teIdx, teVal, teTgt := m0.b200Rows(testSet, m0.autoScale)

	prog := &fmTrialsProgress{ctx: ctx, spans: make([]*monitor.Span, len(trials)), run: make([]int32, len(trials))}
	for k, m := range models {
		_, span := monitor.Start(ctx, "FM.Fit", m.nEpochs)
		defer span.End()
		prog.spans[k] = span
	}
	h := cgo.NewHandle(prog)
	defer h.Delete()

	results := make([]C.gorse_b200_fm_fit_result, len(trials))
	var st C.int32_t
	// the library copies during the call and keeps no Go pointer (cgo rule)
	if len(m0.embeddingDim) == 0 {
		st = C.gorse_b200_fm_fit_trials(c, C.int64_t(m0.numFeatures), C.int32_t(m0.numDimension), C.int32_t(len(trials)), &params[0],
			C.int64_t(trainSet.Count()), &trOff[0], ptrI32(trIdx), ptrF32(trVal), ptrF32(trTgt), nil,
			C.int64_t(testSet.Count()), &teOff[0], ptrI32(teIdx), ptrF32(teVal), ptrF32(teTgt), nil,
			0, nil, 0, nil, nil, (**C.float)(unsafe.Pointer(pin)), C.int64_t(nParams), (**C.float)(unsafe.Pointer(pout)), nil,
			C.gorse_b200_fm_trials_progress_ptr(), unsafe.Pointer(&h), &results[0])
	} else {
		table, rows := b200EmbTable(m0.embeddingDim, trainSet, testSet)
		defer table.free()
		st = C.gorse_b200_fm_fit_trials(c, C.int64_t(m0.numFeatures), C.int32_t(m0.numDimension), C.int32_t(len(trials)), &params[0],
			C.int64_t(trainSet.Count()), &trOff[0], ptrI32(trIdx), ptrF32(trVal), ptrF32(trTgt), &rows[0][0],
			C.int64_t(testSet.Count()), &teOff[0], ptrI32(teIdx), ptrF32(teVal), ptrF32(teTgt), &rows[1][0],
			C.int32_t(len(table.dims)), &table.dims[0], C.int64_t(table.rows), (**C.uint16_t)(unsafe.Pointer(table.slots)), &table.mask[0],
			(**C.float)(unsafe.Pointer(pin)), C.int64_t(nParams), (**C.float)(unsafe.Pointer(pout)), nil,
			C.gorse_b200_fm_trials_progress_ptr(), unsafe.Pointer(&h), &results[0])
	}
	if st == C.GORSE_B200_ERR_UNSUPPORTED {
		log.Logger().Info("gorse_b200 cannot fit these AFM trials; fitting them one by one", zap.Error(afmB200Error(st)))
		return fitTrialsOneByOne(ctx, trials, trainSet, testSet, config), nil
	}
	if err := afmB200Error(st); err != nil {
		return nil, err
	}
	scores := make([]Score, len(trials))
	for k, r := range results {
		if r.cancelled != 0 {
			log.Logger().Info("fit AFM canceled", zap.Error(ctx.Err()))
			continue
		}
		if r.diverged != 0 {
			log.Logger().Warn("model diverged", zap.Float32("lr", models[k].lr))
		}
		scores[k] = Score{Precision: float32(r.precision), Recall: float32(r.recall), Accuracy: float32(r.accuracy), AUC: float32(r.auc)}
	}
	return scores, nil
}

// fitTrialsOneByOne: each trial's own model through (*AFM).Fit, which trains with the reference's fit where the library
// cannot
func fitTrialsOneByOne(ctx context.Context, trials []model.Params, trainSet, testSet dataset.CTRSplit, config *FitConfig) []Score {
	scores := make([]Score, len(trials))
	for k, t := range trials {
		scores[k] = NewAFM(t).Fit(ctx, trainSet, testSet, config)
	}
	return scores
}
