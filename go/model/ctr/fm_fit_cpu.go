// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package model/ctr.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain (see INTEGRATION.md).
// The integration renames the reference's (*AFM).Fit (model/ctr/fm.go:307-417) to fitCPU, so that afm_b200.go can fall
// back to it.  Without the b200 tag this file keeps Fit as it was.

//go:build (!cgo || !xla) && !(b200 && cgo)

package ctr

import (
	"context"

	"github.com/gorse-io/gorse/dataset"
)

// Fit is the reference's AFM.Fit.
func (fm *AFM) Fit(ctx context.Context, trainSet, testSet dataset.CTRSplit, config *FitConfig) Score {
	return fm.fitCPU(ctx, trainSet, testSet, config)
}
