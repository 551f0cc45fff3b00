// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package main of cmd/gorse-bench.
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image).
//
// The integration moves EvaluateAFM's scoring after the fit (main.go:133-206), unchanged, into scoreAFMCPU in main.go,
// which returns the score (INTEGRATION.md, "gorse-bench reranker"), and EvaluateAFM stores scoreAFM's result.  Without the
// tags this file makes scoreAFM the reference's scoring; with them, reranker_b200.go scores on the GPU and falls back to
// scoreAFMCPU.
//go:build !(b200 && cgo && !xla)

package main

import (
	"github.com/gorse-io/gorse/config"
	"github.com/gorse-io/gorse/model/ctr"
)

// scoreAFM is the reference's scoring.
func scoreAFM(cfg *config.Config, ml *ctr.AFM, train, test *ctr.Dataset, exportUserAUC bool) float64 {
	return scoreAFMCPU(cfg, ml, train, test, exportUserAUC)
}
