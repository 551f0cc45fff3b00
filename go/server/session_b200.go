// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package server.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain (see INTEGRATION.md).  The C call behind it,
// (*vectors.B200).SessionRecommend, is mirrored one-to-one by gorse_b200.VectorCollection.session_recommend, which
// tests/test_session_gpu.py drives through the same ABI.
//
// The session recommendation (RestServer.sessionRecommend, rest.go:1069-1173) on the GPU vector store: the loop at
// rest.go:1114-1170 -- one QueryItemToItem and one FilterVisibleItemsByCategories per positive feedback item, up to
// ContextSize of them -- becomes one gorse_b200_vecdb_session_recommend call.  INTEGRATION.md ("Session recommendation")
// shows where the handler calls it.

//go:build b200 && cgo

package server

import (
	"context"
	"errors"
	"strings"

	mapset "github.com/deckarep/golang-set/v2"
	"github.com/gorse-io/gorse/common/expression"
	"github.com/gorse-io/gorse/common/log"
	"github.com/gorse-io/gorse/config"
	"github.com/gorse-io/gorse/storage"
	"github.com/gorse-io/gorse/storage/cache"
	"github.com/gorse-io/gorse/storage/data"
	"github.com/gorse-io/gorse/storage/vectors"
	"github.com/samber/lo"
	"go.uber.org/zap"
)

// sessionRequest is one posted session after the handler's pre-processing: its feedback sorted by data.SortFeedbacks, the
// path's categories and the n / offset query parameters.
type sessionRequest struct {
	Feedback   []data.Feedback
	Categories []string
	N, Offset  int
}

// sessionRecommendB200 answers many session requests of one item-to-item recommender, one library call per distinct
// category list (the item filter is shared by every session of a call).  Row i is what rest.go:1114-1170 followed by the
// offset slice returns for reqs[i].  handled = false: the vector store is not a B200, or the library does not serve these
// arguments (storage.ErrNotSupported); the caller then runs the handler's own loop.
func (s *RestServer) sessionRecommendB200(ctx context.Context, cfg config.ItemToItemConfig, reqs []sessionRequest) ([][]cache.Score, bool, error) {
	store, ok := s.VectorClient.(*vectors.B200)
	if !ok {
		return nil, false, nil
	}
	scoreScale := 1.0
	if cfg.Type == "auto" {
		scoreScale = .5
	}
	groups := map[string][]int{}
	for i, r := range reqs {
		key := strings.Join(r.Categories, "\x00")
		groups[key] = append(groups[key], i)
	}
	results := make([][]cache.Score, len(reqs))
	for _, members := range groups {
		categories := reqs[members[0]].Categories
		contextIds, excludeIds := make([][]string, len(members)), make([][]string, len(members))
		top := 0
		for k, i := range members {
			// rest.go:1110-1121: every item of the session is excluded, the positive ones are the context
			exclude := mapset.NewSet[string]()
			for _, fb := range reqs[i].Feedback {
				exclude.Add(fb.ItemId)
				if expression.MatchFeedbackTypeExpressions(s.Config.Recommend.DataSource.PositiveFeedbackTypes, fb.FeedbackType, fb.Value) {
					contextIds[k] = append(contextIds[k], fb.ItemId)
				}
			}
			excludeIds[k] = exclude.ToSlice()
			top = max(top, reqs[i].N+reqs[i].Offset)
		}
		// FilterVisibleItemsByCategories (rest.go:815-832) for the whole collection, once per call
		itemOK := func(ids []string) ([]bool, error) {
			items, err := s.DataClient.BatchGetItems(ctx, ids, data.GetOptions{})
			if err != nil {
				return nil, err
			}
			visible := mapset.NewSet[string]()
			for _, item := range items {
				if !item.IsHidden && lo.EveryBy(categories, func(c string) bool { return lo.Contains(item.Categories, c) }) {
					visible.Add(item.ItemId)
				}
			}
			return lo.Map(ids, func(id string, _ int) bool { return visible.Contains(id) }), nil
		}
		// the neighbour rows of earlier requests serve this one; answers do not depend on the cache, so the request goes on
		// without it whatever NeighbourCache returns
		if err := store.NeighbourCache(vectors.ItemToItemCollection(cfg.Name), s.Config.Recommend.CacheSize); err != nil &&
			!errors.Is(err, storage.ErrNotSupported) {
			log.Logger().Warn("session recommendation without the neighbour cache", zap.Error(err))
		}
		rows, err := store.SessionRecommend(ctx, vectors.ItemToItemCollection(cfg.Name), contextIds, excludeIds, itemOK,
			s.Config.Recommend.CacheSize, s.Config.Recommend.ContextSize, top, scoreScale)
		if errors.Is(err, storage.ErrNotSupported) {
			return nil, false, nil
		}
		if err != nil {
			return nil, true, err
		}
		// TopKFilter(n + offset) of each request is the first n + offset of the call's `top`; then [offset:][:n]
		for k, i := range members {
			row := rows[k][:min(len(rows[k]), reqs[i].N+reqs[i].Offset)]
			if len(row) > reqs[i].Offset {
				results[i] = row[reqs[i].Offset:]
				results[i] = results[i][:min(len(results[i]), reqs[i].N)]
			}
		}
	}
	return results, true, nil
}
