// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package worker.
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image, see INTEGRATION.md).  Every C call below is mirrored
// one-to-one by gorse_b200.recommend (gorse_b200/__init__.py), which tests/test_recommend_gpu.py drives through the same ABI.
//
// Batched offline recommendation: Pipeline.Recommend (worker/pipeline.go:124-319) for a batch of users in one
// gorse_b200_recommend call.  B200Stages builds the stage list from the RecommendConfig (Ranker.Recommenders, or
// ListRecommenders() when that is empty, as pipeline.go:215-219 does); the worker fills each stage's inputs and calls
// B200Recommend once per batch.  Cold-start users and users without a CF embedding are not sent (pipeline.go:195-213); the
// digest, the categories and timestamps of the results and the LLM ranker stay in Go.
//
// Every array the library reads is copied into C memory first: the stage structs hold pointers, and cgo forbids handing C
// Go memory that contains Go pointers.  The library keeps no pointer after the call, so the copies are freed on return.

//go:build b200 && cgo

package worker

/*
#cgo LDFLAGS: -lgorse_b200
#include <stdlib.h>
#include <string.h>
#include "gorse_b200.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"strings"
	"unsafe"

	"github.com/gorse-io/gorse/common/log"
	"github.com/gorse-io/gorse/config"
	"github.com/gorse-io/gorse/logics"
	"github.com/gorse-io/gorse/storage"
	"github.com/gorse-io/gorse/storage/vectors"
	"go.uber.org/zap"
)

// B200Stage is one recommender of the sequence.  Kind is a gorse_b200_stage_kind; Name is the configured full name.  The
// worker fills the fields of its kind; item ids are indices of the batch's item dictionary.
type B200Stage struct {
	Kind int32
	Name string
	// LIST: one shared list (non-personalized, latest) or one list per user (external, PerUser set)
	ListItems   []int32
	ListScores  []float64
	PerUser     bool
	UserItems   [][]int32
	UserScores  [][]float64
	// ITEM_TO_ITEM / USER_TO_USER: the collection (a *C.gorse_b200_vecdb of storage/vectors, passed as a pointer), CacheSize
	Collection unsafe.Pointer
	N          int32
	ScoreScale float64
	// ITEM_TO_ITEM.  SlotOfItem / ItemOfSlot, and UserSlots / Feedback below, name slots of the collection: a DeleteVectors
	// or Optimize on it renumbers them (gorse_b200_vecdb_compact), so they are built again for every call.
	Context    [][]int32 // per user, positive feedback newest first, -1 = outside the dictionary
	SlotOfItem []int64
	ItemOfSlot []int32
	Categories []int32
	// USER_TO_USER
	UserSlots []int64
	Feedback  [][]int32 // per slot of the collection
	ItemOK    []uint8
}

// B200Stages returns the stage list of the configured recommenders, in order, with Kind and Name set.
func B200Stages(cfg *config.RecommendConfig) ([]B200Stage, error) {
	names := cfg.Ranker.Recommenders
	if len(names) == 0 {
		names = cfg.ListRecommenders()
	}
	stages := make([]B200Stage, 0, len(names))
	for _, name := range names {
		s := B200Stage{Name: name, N: int32(cfg.CacheSize), ScoreScale: 1}
		switch {
		case name == logics.CollaborativeRecommender:
			s.Kind = C.GORSE_B200_STAGE_COLLABORATIVE
		case name == logics.LatestRecommender, strings.HasPrefix(name, logics.NonPersonalizedRecommender):
			s.Kind = C.GORSE_B200_STAGE_LIST
		case strings.HasPrefix(name, logics.ExternalRecommender):
			s.Kind, s.PerUser = C.GORSE_B200_STAGE_LIST, true
		case strings.HasPrefix(name, logics.ItemToItemRecommender):
			s.Kind = C.GORSE_B200_STAGE_ITEM_TO_ITEM
		case strings.HasPrefix(name, logics.UserToUserRecommender):
			s.Kind = C.GORSE_B200_STAGE_USER_TO_USER
		default:
			return nil, fmt.Errorf("unknown recommender: %s", name)
		}
		stages = append(stages, s)
	}
	return stages, nil
}

// B200NeighbourCaches turns on the neighbour cache of every item-to-item and user-to-user stage's collection for the
// stage's N (CacheSize) before B200Recommend, so that the batches of a worker pass reuse the neighbour rows earlier batches
// computed ((*vectors.B200).NeighbourCache).  Call it before every batch: a reload replaces a collection's handle, and with
// an unchanged size the call keeps what the cache holds.  Answers do not depend on the cache, so a stage whose collection
// it cannot serve, or whose sizing fails, runs without it; a failure other than storage.ErrNotSupported is logged.
func B200NeighbourCaches(store *vectors.B200, stages []B200Stage) {
	for _, s := range stages {
		var collection string
		switch s.Kind {
		case C.GORSE_B200_STAGE_ITEM_TO_ITEM:
			collection = vectors.ItemToItemCollection(strings.TrimPrefix(s.Name, logics.ItemToItemRecommender))
		case C.GORSE_B200_STAGE_USER_TO_USER:
			collection = vectors.UserToUserCollection(strings.TrimPrefix(s.Name, logics.UserToUserRecommender))
		default:
			continue
		}
		if err := store.NeighbourCache(collection, int(s.N)); err != nil && !errors.Is(err, storage.ErrNotSupported) {
			log.Logger().Warn("recommender without the neighbour cache", zap.String("recommender", s.Name), zap.Error(err))
		}
	}
}

// B200CF is the CF recall input (updateCollaborativeRecommend, pipeline.go:403-449).
type B200CF struct {
	Collection  unsafe.Pointer // *C.gorse_b200_vecdb of the "collaborative_filtering_<id>" collection
	UserVectors []float32      // n_users x dim
	SlotOfItem  []int64        // like the stages' maps, stale after a DeleteVectors or Optimize on the collection
	ItemOfSlot  []int32
	N           int32
}

// B200Ranker is the FM ranker input: the handle of model/ctr.AFMB200 and the factored rows gorse_b200_fm_rank takes.
type B200Ranker struct {
	FM                                   unsafe.Pointer // *C.gorse_b200_fm
	UserFeat, ItemFeat                   []int32
	UserLabOff, ItemLabOff               []int64
	UserLabIdx, ItemLabIdx               []int32
	UserLabVal, ItemLabVal               []float32
	ItemEmb                              [][]uint16 // per slot, n_items x dim bf16 bits
	ItemEmbMask                          []uint8
}

// cArena copies Go slices into C memory and frees them together.
type cArena struct{ ptrs []unsafe.Pointer }

func (a *cArena) copy(p unsafe.Pointer, bytes int) unsafe.Pointer {
	if bytes == 0 {
		return nil
	}
	c := C.malloc(C.size_t(bytes))
	C.memcpy(c, p, C.size_t(bytes))
	a.ptrs = append(a.ptrs, c)
	return c
}

func (a *cArena) i32(s []int32) *C.int32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int32_t)(a.copy(unsafe.Pointer(&s[0]), 4*len(s)))
}

func (a *cArena) i64(s []int64) *C.int64_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int64_t)(a.copy(unsafe.Pointer(&s[0]), 8*len(s)))
}

func (a *cArena) f32(s []float32) *C.float {
	if len(s) == 0 {
		return nil
	}
	return (*C.float)(a.copy(unsafe.Pointer(&s[0]), 4*len(s)))
}

func (a *cArena) f64(s []float64) *C.double {
	if len(s) == 0 {
		return nil
	}
	return (*C.double)(a.copy(unsafe.Pointer(&s[0]), 8*len(s)))
}

func (a *cArena) u8(s []uint8) *C.uint8_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint8_t)(a.copy(unsafe.Pointer(&s[0]), len(s)))
}

func (a *cArena) free() {
	for _, p := range a.ptrs {
		C.free(p)
	}
	a.ptrs = nil
}

// csr flattens per-row lists into offsets from 0 and entries
func csrI32(rows [][]int32) ([]int64, []int32) {
	off := make([]int64, len(rows)+1)
	flat := make([]int32, 0)
	for i, r := range rows {
		flat = append(flat, r...)
		off[i+1] = int64(len(flat))
	}
	return off, flat
}

func csrF64(rows [][]float64) []float64 {
	flat := make([]float64, 0)
	for _, r := range rows {
		flat = append(flat, r...)
	}
	return flat
}

// B200Recommend runs gorse_b200_recommend for one batch.  exclude[u]: the user's feedback items (-1 = outside the
// dictionary); live[n_items]; cf and ranker may be nil; replacement (ranked calls only) holds each user's distinct
// positive / read feedback items.  Returns each user's items and scores: ranked by the FM, or the merged candidates.
func B200Recommend(ctx unsafe.Pointer, exclude [][]int32, nItems int, live []uint8, stages []B200Stage, cf *B200CF, ranker *B200Ranker,
	replItems [][]int32, replPositive [][]uint8, positiveDecay, readDecay float64) ([][]int32, [][]float64, error) {
	var a cArena
	defer a.free()
	nUsers := len(exclude)
	eOff, eItems := csrI32(exclude)
	bound := make([]int64, nUsers)
	cs := (*[1 << 16]C.gorse_b200_recommend_stage)(C.calloc(C.size_t(len(stages)+1), C.size_t(unsafe.Sizeof(C.gorse_b200_recommend_stage{}))))
	a.ptrs = append(a.ptrs, unsafe.Pointer(cs))
	for i, s := range stages {
		d := &cs[i]
		d.kind = C.int32_t(s.Kind)
		switch s.Kind {
		case C.GORSE_B200_STAGE_LIST:
			if s.PerUser {
				off, items := csrI32(s.UserItems)
				d.list_off, d.list_items, d.list_scores = a.i64(off), a.i32(items), a.f64(csrF64(s.UserScores))
				for u := range bound {
					bound[u] += int64(len(s.UserItems[u]))
				}
			} else {
				d.list_len, d.list_items, d.list_scores = C.int64_t(len(s.ListItems)), a.i32(s.ListItems), a.f64(s.ListScores)
				for u := range bound {
					bound[u] += int64(len(s.ListItems))
				}
			}
		case C.GORSE_B200_STAGE_COLLABORATIVE:
			if cf != nil {
				for u := range bound {
					bound[u] += int64(cf.N)
				}
			}
		default:
			d.db, d.n, d.score_scale = (*C.gorse_b200_vecdb)(s.Collection), C.int32_t(s.N), C.double(s.ScoreScale)
			for u := range bound {
				bound[u] += int64(s.N)
			}
			if s.Kind == C.GORSE_B200_STAGE_ITEM_TO_ITEM {
				off, items := csrI32(s.Context)
				d.ctx_off, d.ctx_items = a.i64(off), a.i32(items)
				d.slot_of_item, d.item_of_slot = a.i64(s.SlotOfItem), a.i32(s.ItemOfSlot)
				d.categories, d.n_categories = a.i32(s.Categories), C.int32_t(len(s.Categories))
			} else {
				off, items := csrI32(s.Feedback)
				d.user_slots, d.n_fb_rows = a.i64(s.UserSlots), C.int64_t(len(s.Feedback))
				d.fb_off, d.fb_items, d.item_ok = a.i64(off), a.i32(items), a.u8(s.ItemOK)
			}
		}
	}
	var ccf *C.gorse_b200_recommend_cf
	if cf != nil {
		ccf = (*C.gorse_b200_recommend_cf)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gorse_b200_recommend_cf{}))))
		a.ptrs = append(a.ptrs, unsafe.Pointer(ccf))
		ccf.db, ccf.user_vectors = (*C.gorse_b200_vecdb)(cf.Collection), a.f32(cf.UserVectors)
		ccf.slot_of_item, ccf.item_of_slot, ccf.n = a.i64(cf.SlotOfItem), a.i32(cf.ItemOfSlot), C.int32_t(cf.N)
	}
	var crk *C.gorse_b200_recommend_ranker
	var rOff []int64
	var rItems []int32
	var rPos []uint8
	if ranker != nil {
		crk = (*C.gorse_b200_recommend_ranker)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gorse_b200_recommend_ranker{}))))
		a.ptrs = append(a.ptrs, unsafe.Pointer(crk))
		crk.fm = (*C.gorse_b200_fm)(ranker.FM)
		crk.user_feat, crk.user_lab_off, crk.user_lab_idx, crk.user_lab_val = a.i32(ranker.UserFeat), a.i64(ranker.UserLabOff), a.i32(ranker.UserLabIdx), a.f32(ranker.UserLabVal)
		crk.item_feat, crk.item_lab_off, crk.item_lab_idx, crk.item_lab_val = a.i32(ranker.ItemFeat), a.i64(ranker.ItemLabOff), a.i32(ranker.ItemLabIdx), a.f32(ranker.ItemLabVal)
		if len(ranker.ItemEmb) > 0 {
			embs := (*[64]*C.uint16_t)(C.calloc(C.size_t(len(ranker.ItemEmb)), C.size_t(unsafe.Sizeof(uintptr(0)))))
			a.ptrs = append(a.ptrs, unsafe.Pointer(embs))
			for s, e := range ranker.ItemEmb {
				if len(e) > 0 {
					embs[s] = (*C.uint16_t)(a.copy(unsafe.Pointer(&e[0]), 2*len(e)))
				}
			}
			crk.item_emb = (**C.uint16_t)(unsafe.Pointer(embs))
		}
		crk.item_emb_mask = a.u8(ranker.ItemEmbMask)
		if replItems != nil {
			rOff, rItems = csrI32(replItems)
			for u := range bound {
				bound[u] += int64(len(replItems[u]))
				rPos = append(rPos, replPositive[u]...)
			}
		}
	}
	total := int64(0)
	for _, b := range bound {
		total += b
	}
	outItems := (*C.int32_t)(C.calloc(C.size_t(total+1), 4))
	outScores := (*C.double)(C.calloc(C.size_t(total+1), 8))
	counts := (*C.int32_t)(C.calloc(C.size_t(nUsers+1), 4))
	a.ptrs = append(a.ptrs, unsafe.Pointer(outItems), unsafe.Pointer(outScores), unsafe.Pointer(counts))
	st := C.gorse_b200_recommend((*C.gorse_b200_ctx)(ctx), C.int64_t(nUsers), a.i64(eOff), a.i32(eItems), C.int32_t(nItems), a.u8(live),
		C.int32_t(len(stages)), &cs[0], ccf, crk, a.i64(rOff), a.i32(rItems), a.u8(rPos), C.double(positiveDecay), C.double(readDecay),
		outItems, outScores, counts, nil)
	if st != C.GORSE_B200_OK {
		return nil, nil, fmt.Errorf("gorse_b200_recommend: status %d: %s", int(st), C.GoString(C.gorse_b200_last_error()))
	}
	items := unsafe.Slice((*int32)(unsafe.Pointer(outItems)), total+1)
	scores := unsafe.Slice((*float64)(unsafe.Pointer(outScores)), total+1)
	cnt := unsafe.Slice((*int32)(unsafe.Pointer(counts)), nUsers+1)
	resItems, resScores := make([][]int32, nUsers), make([][]float64, nUsers)
	at := int64(0)
	for u := 0; u < nUsers; u++ {
		c := int64(cnt[u])
		resItems[u] = append([]int32(nil), items[at:at+c]...)     // copied out before the arena frees the C buffers
		resScores[u] = append([]float64(nil), scores[at:at+c]...)
		at += bound[u]
	}
	return resItems, resScores, nil
}
