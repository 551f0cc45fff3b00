// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package main of cmd/gorse-bench.
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image).
//
// The integration moves the per-user loop and the averaging of EvaluateEmbedding (main.go:403-465), unchanged, into
// scoreEmbeddingsCPU in main.go, which returns the score (INTEGRATION.md, "gorse-bench embedding"), and EvaluateEmbedding
// calls scoreEmbeddings.  Without the b200 tag this file makes scoreEmbeddings the reference's loop, parallel over `jobs`
// as before; with it, embedding_b200.go scores on the GPU and falls back to scoreEmbeddingsCPU.
//go:build !(b200 && cgo)

package main

import (
	"github.com/gorse-io/gorse/dataset"
	"github.com/gorse-io/gorse/model/cf"
)

// scoreEmbeddings is the reference's scoring.
func scoreEmbeddings(train, test dataset.CFSplit, embeddings [][]float32, topK, jobs int) cf.Score {
	return scoreEmbeddingsCPU(train, test, embeddings, topK, jobs)
}
