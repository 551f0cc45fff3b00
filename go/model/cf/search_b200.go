//go:build b200 && cgo

package cf

/*
#include "gorse_b200.h"

// the per-epoch callback of gorse_b200_cf_fit_trials goes through this exported trampoline (see b200.go)
extern int32_t gorseB200TrialsProgress(void *user, int32_t epoch, int32_t nTrials, gorse_b200_trial_state *states);
static int32_t gorse_b200_trials_progress_tramp(void *user, int32_t epoch, int32_t n, const gorse_b200_trial_state *states) {
    return gorseB200TrialsProgress(user, epoch, n, (gorse_b200_trial_state *)states);
}
static gorse_b200_trials_progress_fn gorse_b200_trials_progress_ptr(void) { return gorse_b200_trials_progress_tramp; }
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

// SearchTrial is one trial of optimizeCollaborativeFiltering (master/tasks.go:1268-1316): the model type ModelSearch
// suggested ("BPR" or "ALS") and the parameters of that type's SuggestParams (model/cf/model.go:397-405, 588-596).
type SearchTrial struct {
	Type   string
	Params model.Params
}

type trialsProgress struct {
	ctx   context.Context
	spans []*monitor.Span
	run   []int32
}

//export gorseB200TrialsProgress
func gorseB200TrialsProgress(user unsafe.Pointer, epoch, nTrials C.int32_t, states *C.gorse_b200_trial_state) C.int32_t {
	p := (*(*cgo.Handle)(user)).Value().(*trialsProgress)
	for k := 0; k < int(nTrials); k++ {
		s := (*C.gorse_b200_trial_state)(unsafe.Add(unsafe.Pointer(states), uintptr(k)*unsafe.Sizeof(*states)))
		for ; p.run[k] < int32(s.epochs_run); p.run[k]++ {
			p.spans[k].Add(1) // model/cf/model.go:519, once per epoch of each trial
		}
	}
	if p.ctx.Err() != nil {
		return 1 // unfinished trials return Score{} (:491-493)
	}
	return 0
}

// FitTrialsB200 fits the trials in one gorse_b200_cf_fit_trials call and returns their scores in trial order: trial k's
// score is what m.Fit(ctx, trainSet, valSet, config) returns for m = the trial's model with its parameters set, which is
// what ModelSearch.Objective (model/cf/optimize.go:61-81) compares.  The models are discarded, as the reference discards
// the search's models; the master re-fits the winner (master/tasks.go:897-921).  An error means no trial was fitted.
func FitTrialsB200(ctx context.Context, trials []SearchTrial, trainSet, valSet dataset.CFSplit, config *FitConfig) ([]Score, error) {
	if len(trials) == 0 {
		return nil, nil
	}
	c, err := b200Context()
	if err != nil {
		return nil, err
	}
	params := make([]C.gorse_b200_fit_params, len(trials))
	als := make([]int32, len(trials))
	for k, t := range trials {
		p := &params[k]
		switch t.Type {
		case "BPR":
			m := NewBPR(t.Params)
			C.gorse_b200_fit_params_default(0, p)
			p.n_factors, p.n_epochs = C.int32_t(m.nFactors), C.int32_t(m.nEpochs)
			p.lr, p.reg = C.float(m.lr), C.float(m.reg)
			p.init_mean, p.init_stddev = C.float(m.initMean), C.float(m.initStdDev)
			p.seed = C.uint64_t(m.GetRandomGenerator().Int63())
		case "ALS":
			m := NewALS(t.Params)
			als[k] = 1
			C.gorse_b200_fit_params_default(1, p)
			p.n_factors, p.n_epochs = C.int32_t(m.nFactors), C.int32_t(m.nEpochs)
			p.reg, p.alpha = C.float(m.reg), C.float(m.weight)
			p.init_mean, p.init_stddev = C.float(m.initMean), C.float(m.initStdDev)
			p.seed = C.uint64_t(m.GetRandomGenerator().Int63())
		default:
			return nil, errors.New("unknown model type " + t.Type)
		}
		p.verbose, p.candidates = C.int32_t(config.Verbose), C.int32_t(config.Candidates)
		p.topk, p.patience = C.int32_t(config.TopK), C.int32_t(config.Patience)
	}
	nUsers, nItems, d := trainSet.CountUsers(), trainSet.CountItems(), int(params[0].n_factors)
	uOff, uIdx := flattenCSR(trainSet.GetUserFeedback())
	iOff, iIdx := flattenCSR(trainSet.GetItemFeedback())
	tOff, tIdx := flattenCSR(valSet.GetUserFeedback())

	var cf *C.gorse_b200_cf
	if err := b200Error(C.gorse_b200_cf_create(c, C.int32_t(nUsers), C.int32_t(nItems), C.int32_t(d),
		i64ptr(uOff), i32ptr(uIdx), i64ptr(iOff), i32ptr(iIdx), &cf)); err != nil {
		return nil, err
	}
	defer C.gorse_b200_cf_destroy(cf)

	prog := &trialsProgress{ctx: ctx, spans: make([]*monitor.Span, len(trials)), run: make([]int32, len(trials))}
	for k, t := range trials {
		_, span := monitor.Start(ctx, t.Type+".Fit", int(params[k].n_epochs)) // :442 / :639
		defer span.End()
		prog.spans[k] = span
	}
	h := cgo.NewHandle(prog)
	defer h.Delete()

	results := make([]C.gorse_b200_fit_result, len(trials))
	// the library copies during the call and keeps no Go pointer (cgo rule)
	if err := b200Error(C.gorse_b200_cf_fit_trials(cf, C.int32_t(len(trials)), (*C.int32_t)(unsafe.Pointer(&als[0])), &params[0],
		i64ptr(tOff), i32ptr(tIdx), nil, nil, C.gorse_b200_trials_progress_ptr(), unsafe.Pointer(&h), &results[0], nil, nil)); err != nil {
		return nil, err
	}
	scores := make([]Score, len(trials))
	for k, r := range results {
		if r.cancelled != 0 {
			log.Logger().Info("fit canceled", zap.String("type", trials[k].Type), zap.Int("epoch", int(r.epochs_run)))
			continue
		}
		scores[k] = Score{NDCG: float32(r.ndcg), Precision: float32(r.precision), Recall: float32(r.recall)}
	}
	return scores, nil
}
