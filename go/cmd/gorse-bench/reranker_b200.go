// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package main of cmd/gorse-bench.
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image).  The C call it makes, through (*ctr.AFM).GAUCB200
// (go/model/ctr/gauc_b200.go), is mirrored one-to-one by the ctypes binding gorse_b200.ranker_gauc, which the GPU
// test-suite exercises.
//
// scoreAFM on the GPU: `gorse-bench reranker`'s AFM scoring after the fit (EvaluateAFM, main.go:133-206) in one
// gorse_b200_fm_gauc call.  INTEGRATION.md ("gorse-bench reranker") shows the edit that calls this function and moves the
// reference's scoring, unchanged, into scoreAFMCPU.  Built without the tags, reranker_cpu.go makes that scoring scoreAFM.
//go:build b200 && cgo && !xla

package main

import (
	"encoding/csv"
	"fmt"
	"os"
	"strconv"

	"github.com/gorse-io/gorse/common/log"
	"github.com/gorse-io/gorse/config"
	"github.com/gorse-io/gorse/model/ctr"
	"go.uber.org/zap"
)

// scoreAFM counts every user's positive training rows as the reference does, makes one call, and writes AFM.csv from the
// per-user rows it returns, in ascending user order.  A library error is logged and the reference's scoring runs instead.
func scoreAFM(cfg *config.Config, ml *ctr.AFM, train, test *ctr.Dataset, exportUserAUC bool) float64 {
	nUsers := 0
	for _, set := range []*ctr.Dataset{train, test} {
		for i := 0; i < set.Count(); i++ {
			indices, _, _, _ := set.Get(i)
			if len(indices) > 0 && int(indices[0]) >= nUsers {
				nUsers = int(indices[0]) + 1
			}
		}
	}
	feedbackCount := make([]int64, nUsers)
	for i := 0; i < train.Count(); i++ {
		indices, _, _, target := train.Get(i)
		if target > 0 {
			feedbackCount[indices[0]]++
		}
	}
	score, users, err := ml.GAUCB200(test, feedbackCount, cfg.Recommend.ContextSize)
	if err != nil {
		log.Logger().Error("gorse_b200_fm_gauc failed; scoring on the CPU", zap.Error(err))
		return scoreAFMCPU(cfg, ml, train, test, exportUserAUC)
	}
	if exportUserAUC {
		csvFile, err := os.Create("AFM.csv")
		if err != nil {
			log.Logger().Error("failed to create AFM.csv", zap.Error(err))
			return score
		}
		defer csvFile.Close()
		csvWriter := csv.NewWriter(csvFile)
		defer csvWriter.Flush()
		_ = csvWriter.Write([]string{"Feedback", "Candidates", "AUC"})
		for _, u := range users {
			_ = csvWriter.Write([]string{strconv.Itoa(u.Feedback), strconv.Itoa(u.Candidates), fmt.Sprintf("%.4f", u.AUC)})
		}
	}
	return score
}
