// Copyright 2026 gorse-b200 authors. Drop-in for gorse-io/gorse @ 5404aefa, package storage/vectors.
//
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image, see INTEGRATION.md).  Every C call below is mirrored
// one-to-one by gorse_b200.VectorCollection (gorse_b200/__init__.py), which tests/test_vecdb_gpu.py drives through the same
// ABI on the reference's own test values (storage/vectors/database_test.go).
//
// A vectors.Database (database.go:107-120) whose collections live in GPU memory: item-to-item, user-to-user and CF retrieval
// reach it with NO change to master / worker / logics -- set `database.vector_store = "b200://0"` (device ordinal) and the
// init() below makes vectors.Open (database.go:168-175) return it.  The library works on slots and int32 category ids; this
// file owns the id <-> slot and category string <-> id maps, which is all the reference's backends keep on the host too.
//
// "b200://<device>/<root>" also keeps every collection in <root>/<tablePrefix><name>.b200vec (root is an absolute path:
// "b200://0/var/lib/gorse/vectors"), so that the master's collections reach a worker and a server that open the same URL on
// a volume all of them mount, and survive a restart.  The process that writes a collection saves it; every process reloads a
// collection whose file carries a newer generation before it reads it.  See INTEGRATION.md.

//go:build b200 && cgo

package vectors

/*
#cgo LDFLAGS: -lgorse_b200
#include <stdlib.h>
#include "gorse_b200.h"

// cgo cannot call Go closures from C directly: the snapshot stream goes through these exported trampolines.
extern int32_t gorseB200SnapshotWrite(void *user, void *buf, int64_t n);
extern int64_t gorseB200SnapshotRead(void *user, void *buf, int64_t n);
static int32_t gorse_b200_snapshot_write_tramp(void *user, const void *buf, int64_t n) { return gorseB200SnapshotWrite(user, (void *)buf, n); }
static int64_t gorse_b200_snapshot_read_tramp(void *user, void *buf, int64_t n) { return gorseB200SnapshotRead(user, buf, n); }
static gorse_b200_write_fn gorse_b200_snapshot_write_ptr(void) { return gorse_b200_snapshot_write_tramp; }
static gorse_b200_read_fn gorse_b200_snapshot_read_ptr(void) { return gorse_b200_snapshot_read_tramp; }
*/
import "C"

import (
	"bufio"
	"context"
	"encoding/binary"
	"fmt"
	"io"
	"net/url"
	"os"
	"path/filepath"
	"runtime"
	"runtime/cgo"
	"sort"
	"strconv"
	"strings"
	"sync"
	"time"
	"unsafe"

	"github.com/gorse-io/gorse/common/log"
	"github.com/gorse-io/gorse/storage"
	"github.com/gorse-io/gorse/storage/cache"
	"github.com/juju/errors"
	"go.uber.org/zap"
)

const b200Prefix = "b200://"

// the device memory one collection's neighbour cache may take unless the URL sets neighbour_cache_mb
const b200NeighbourCacheMB = 1024

func init() {
	Register([]string{b200Prefix}, func(path, tablePrefix string, opts ...storage.Option) (Database, error) {
		// b200://<device>[/<root>][?neighbour_cache_mb=<MB>&neighbour_fill_n=<n>]
		path, query, _ := strings.Cut(path, "?")
		dev, root, _ := strings.Cut(strings.TrimPrefix(path, b200Prefix), "/")
		device, err := strconv.Atoi(dev)
		if err != nil {
			device = 0
		}
		if root != "" {
			root = "/" + root
		}
		cacheMB := int64(b200NeighbourCacheMB)
		q, err := url.ParseQuery(query)
		if err != nil {
			return nil, errors.Annotatef(err, "b200 store URL %q", path)
		}
		if q.Has("neighbour_cache_mb") {
			// a typo must not leave the default budget in place: anything but a whole number of MB in [0, 2^30] is refused
			mb, err := strconv.ParseInt(q.Get("neighbour_cache_mb"), 10, 64)
			if err != nil || mb < 0 || mb > 1<<30 {
				return nil, errors.Errorf("b200 store URL: neighbour_cache_mb = %q is not a number of MB in [0, 2^30] (0 turns the cache off)",
					q.Get("neighbour_cache_mb"))
			}
			cacheMB = mb
		}
		fillN := 0
		if q.Has("neighbour_fill_n") {
			n, err := strconv.Atoi(q.Get("neighbour_fill_n"))
			if err != nil || n < 0 || n > 1024 {
				return nil, errors.Errorf("b200 store URL: neighbour_fill_n = %q is not an n in [0, 1024] (0 turns the fill off)",
					q.Get("neighbour_fill_n"))
			}
			fillN = n
		}
		return &B200{device: device, tablePrefix: tablePrefix, root: root, cacheMB: cacheMB, fillN: fillN,
			collections: map[string]*b200Collection{}}, nil
	})
}

type b200Collection struct {
	info    CollectionInfo
	handle  *C.gorse_b200_vecdb
	slotOf  map[string]int64 // id -> live slot
	idOf    []string         // slot -> id
	catsOf  [][]string       // slot -> categories (returned with query results, xvec.go:428-430)
	catID   map[string]int32
	catName []string
	// with a root: the generation and the stat of the file last saved or loaded (generation 0: none yet), and writes not
	// yet saved
	generation int64
	file       os.FileInfo
	dirty      bool
	lastWrite  time.Time
	// the neighbour lists saved with this generation (<file>.nbr) are loaded at most once into this handle
	nbrOnce sync.Once
}

// B200 implements Database on one GPU.
type B200 struct {
	mu          sync.RWMutex
	device      int
	tablePrefix string
	root        string // "" = nothing is kept on disk
	cacheMB     int64  // neighbour cache budget per collection, MB (0 = off)
	fillN       int    // with a root: the n at which the writing process fills and saves neighbour lists (0 = off)
	ctx         *C.gorse_b200_ctx
	collections map[string]*b200Collection
	stop        chan struct{}
	flusher     sync.WaitGroup
}

var _ Database = (*B200)(nil)

func b200Err(st C.int32_t) error {
	if st == C.GORSE_B200_OK {
		return nil
	}
	return errors.New(C.GoString(C.gorse_b200_last_error()))
}

// Init opens the device and, with a root, loads every <root>/<tablePrefix><name>.b200vec, as xvec's Init opens its
// directories (xvec.go:60-123), and starts the flusher that saves collections 5 s after their last write.
func (db *B200) Init() error {
	db.mu.Lock()
	defer db.mu.Unlock()
	if db.ctx != nil {
		return nil
	}
	if err := b200Err(C.gorse_b200_ctx_create(C.int32_t(db.device), &db.ctx)); err != nil {
		return err
	}
	if db.root == "" {
		return nil
	}
	if err := os.MkdirAll(db.root, 0o755); err != nil {
		return errors.Trace(err)
	}
	files, err := filepath.Glob(filepath.Join(db.root, db.tablePrefix+"*"+b200FileSuffix))
	if err != nil {
		return errors.Trace(err)
	}
	for _, f := range files {
		name := strings.TrimSuffix(strings.TrimPrefix(filepath.Base(f), db.tablePrefix), b200FileSuffix)
		if err := db.reload(name); err != nil {
			return err
		}
	}
	db.stop = make(chan struct{})
	db.flusher.Add(1)
	go db.flush()
	return nil
}

// Optimize reclaims the slots of deleted vectors (xvec.go:125-131 optimizes its index here): the live vectors keep their
// order in slots 0 .. live-1.  Slot maps taken from this collection before the call are stale afterwards.
func (db *B200) Optimize(ctx context.Context, name string) error {
	db.mu.Lock()
	defer db.mu.Unlock()
	c, err := db.collection(name)
	if err != nil {
		return err
	}
	if err := c.compact(); err != nil {
		return err
	}
	return db.save(name, c)
}

// compact runs gorse_b200_vecdb_compact and renames slotOf, idOf and catsOf through its map; the caller holds db.mu for
// writing.
func (c *b200Collection) compact() error {
	if len(c.idOf) == 0 {
		return nil
	}
	newSlot := make([]int64, len(c.idOf))
	if err := b200Err(C.gorse_b200_vecdb_compact(c.handle, i64p(newSlot), nil)); err != nil {
		return err
	}
	idOf, catsOf := make([]string, 0, len(c.slotOf)), make([][]string, 0, len(c.slotOf))
	for old, slot := range newSlot {
		if slot >= 0 {
			idOf, catsOf = append(idOf, c.idOf[old]), append(catsOf, c.catsOf[old])
		}
	}
	for id, old := range c.slotOf {
		c.slotOf[id] = newSlot[old]
	}
	c.idOf, c.catsOf = idOf, catsOf
	return nil
}

func (db *B200) Close() error {
	if db.stop != nil {
		close(db.stop)
		db.flusher.Wait()
		db.stop = nil
	}
	db.mu.Lock()
	defer db.mu.Unlock()
	var saveErr error
	for name, c := range db.collections {
		if err := db.save(name, c); err != nil && saveErr == nil {
			saveErr = err
		}
		C.gorse_b200_vecdb_destroy(c.handle)
		delete(db.collections, name)
	}
	if db.ctx != nil {
		C.gorse_b200_ctx_destroy(db.ctx)
		db.ctx = nil
	}
	return saveErr
}

func (db *B200) ListCollections(ctx context.Context) ([]string, error) {
	if db.root != "" { // the collections another process saved
		files, err := filepath.Glob(filepath.Join(db.root, db.tablePrefix+"*"+b200FileSuffix))
		if err != nil {
			return nil, errors.Trace(err)
		}
		names := map[string]struct{}{}
		for _, f := range files {
			names[strings.TrimSuffix(strings.TrimPrefix(filepath.Base(f), db.tablePrefix), b200FileSuffix)] = struct{}{}
		}
		db.mu.RLock()
		for name := range db.collections { // and the ones whose file was removed: refresh forgets them
			names[name] = struct{}{}
		}
		db.mu.RUnlock()
		for name := range names {
			if err := db.refresh(name); err != nil {
				return nil, err
			}
		}
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	names := make([]string, 0, len(db.collections))
	for name := range db.collections {
		names = append(names, name)
	}
	sort.Strings(names)
	return names, nil
}

func (db *B200) collection(name string) (*b200Collection, error) {
	c, ok := db.collections[name]
	if !ok {
		return nil, fmt.Errorf("collection %s: %w", name, storage.ErrNotFound)
	}
	return c, nil
}

func (db *B200) DescribeCollection(ctx context.Context, name string) (*CollectionInfo, error) {
	if err := db.refresh(name); err != nil {
		return nil, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(name)
	if err != nil {
		return nil, err
	}
	info := c.info
	return &info, nil
}

func (db *B200) AddCollection(ctx context.Context, name string, dimensions int, distance Distance, config VectorConfig) error {
	if config.Type != QuantizationNone {
		return fmt.Errorf("quantization type %s for b200 %w", config.Type, storage.ErrNotSupported)
	}
	db.mu.Lock()
	defer db.mu.Unlock()
	if _, exists := db.collections[name]; exists {
		return errors.Errorf("collection %s already exists", name)
	}
	c := &b200Collection{info: CollectionInfo{Name: name, Dimension: dimensions, Distance: distance},
		slotOf: map[string]int64{}, catID: map[string]int32{}}
	// vectors.Distance and gorse_b200_distance share their numbering (database.go:27-33)
	if err := b200Err(C.gorse_b200_vecdb_create(db.ctx, C.int32_t(dimensions), C.int32_t(distance), &c.handle)); err != nil {
		return err
	}
	db.collections[name] = c
	c.touch()
	return nil
}

func (db *B200) DeleteCollection(ctx context.Context, name string) error {
	db.mu.Lock()
	defer db.mu.Unlock()
	c, err := db.collection(name)
	if err != nil {
		return err
	}
	delete(db.collections, name)
	if db.root != "" {
		if err := os.Remove(db.path(name)); err != nil && !os.IsNotExist(err) {
			return errors.Trace(err)
		}
		if err := os.Remove(db.path(name) + b200NbrSuffix); err != nil && !os.IsNotExist(err) {
			return errors.Trace(err)
		}
	}
	return b200Err(C.gorse_b200_vecdb_destroy(c.handle))
}

func (db *B200) CountVectors(ctx context.Context, name string) (int64, error) {
	if err := db.refresh(name); err != nil {
		return 0, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(name)
	if err != nil {
		return 0, err
	}
	var live C.int64_t
	if err := b200Err(C.gorse_b200_vecdb_count(c.handle, &live, nil)); err != nil {
		return 0, err
	}
	return int64(live), nil
}

// AddVectors is an upsert by id (xvec.go:288-318): one flat upload per call.
func (db *B200) AddVectors(ctx context.Context, name string, vectors []Vector) error {
	if len(vectors) == 0 {
		return nil
	}
	db.mu.Lock()
	defer db.mu.Unlock()
	c, err := db.collection(name)
	if err != nil {
		return err
	}
	n, dim := len(vectors), c.info.Dimension
	var values []float32
	var spOff []int64
	var spIdx []uint32
	if dim == 0 {
		spOff = make([]int64, n+1)
	}
	hidden, ts, replace := make([]uint8, n), make([]int64, n), make([]int64, n)
	catOff, cats := make([]int64, n+1), []int32{}
	seen := map[string]int{}
	for i, v := range vectors {
		if dim > 0 {
			if len(v.Values) != dim {
				return errors.Errorf("vector %s has dimension %d, want %d", v.Id, len(v.Values), dim)
			}
			values = append(values, v.Values...)
		} else {
			values, spIdx = append(values, v.Values...), append(spIdx, v.Indices...)
			spOff[i+1] = int64(len(spIdx))
		}
		if v.IsHidden {
			hidden[i] = 1
		}
		ts[i] = v.Timestamp.UnixMilli()
		for _, cat := range v.Categories {
			id, ok := c.catID[cat]
			if !ok {
				id = int32(len(c.catName))
				c.catID[cat], c.catName = id, append(c.catName, cat)
			}
			cats = append(cats, id)
		}
		catOff[i+1] = int64(len(cats))
		replace[i] = -1
		if old, ok := c.slotOf[v.Id]; ok {
			replace[i] = old
		}
		if j, dup := seen[v.Id]; dup { // the same id twice in one call: the later one wins, like an upsert
			hidden[j] = 1
		}
		seen[v.Id] = i
	}
	var first C.int64_t
	st := C.gorse_b200_vecdb_add(c.handle, C.int64_t(n), f32p(values), i64p(spOff), u32p(spIdx), u8p(hidden), i64p(ts),
		i64p(catOff), i32p(cats), i64p(replace), &first)
	runtime.KeepAlive(values)
	if err := b200Err(st); err != nil {
		return err
	}
	for i, v := range vectors {
		c.slotOf[v.Id] = int64(first) + int64(i)
		c.idOf = append(c.idOf, v.Id)
		c.catsOf = append(c.catsOf, v.Categories)
	}
	c.touch()
	return nil
}

// AddIDFVectors is the master's rewrite of a sparse item-to-item or user-to-user collection (updateItemToItem /
// updateUserToUser, master/tasks.go:783-877) with the vectors built on the device: row i's vector is appendSparseVector of
// its sorted tag ids over tagsIDF, then of its sorted feedback ids over feedbackIDF at offset len(tagsIDF)
// (logics/item_to_item.go:205-247, logics/user_to_user.go:194-237).  "users" and "items" pass feedback only (tags nil),
// "tags" passes tags only, "auto" passes both.  An id repeated within one row's tags or feedback is kept once.  A row whose
// vector is empty is not added, as VectorWriter.Add drops it (logics/vector_writer.go:84-92): its id keeps its previous
// vector until DeleteVectors.  Otherwise an upsert by id, like AddVectors; an id may appear once per call.
func (db *B200) AddIDFVectors(ctx context.Context, name string, ids []string, hidden []bool, categories [][]string, timestamp time.Time,
	tags [][]int32, tagsIDF []float32, feedback [][]int32, feedbackIDF []float32) error {
	n := len(ids)
	if n == 0 {
		return nil
	}
	if len(hidden) != n || len(categories) != n {
		return errors.Errorf("%d ids with %d hidden flags and %d category lists", n, len(hidden), len(categories))
	}
	if (tags == nil && feedback == nil) || (tags != nil && len(tags) != n) || (feedback != nil && len(feedback) != n) {
		return errors.Errorf("%d ids need %d rows of tags and/or feedback", n, n)
	}
	db.mu.Lock()
	defer db.mu.Unlock()
	c, err := db.collection(name)
	if err != nil {
		return err
	}
	aRows, aIDF, bRows, bIDF := tags, tagsIDF, feedback, feedbackIDF
	if tags == nil {
		aRows, aIDF, bRows, bIDF = feedback, feedbackIDF, nil, nil
	}
	aOff, aIDs := flattenCSR(aRows)
	var bOff []int64
	var bIDs []int32
	if bRows != nil {
		bOff, bIDs = flattenCSR(bRows)
	}
	hid, replace := make([]uint8, n), make([]int64, n)
	catOff, cats := make([]int64, n+1), []int32{}
	seen := make(map[string]struct{}, n)
	for i, id := range ids {
		if _, dup := seen[id]; dup {
			return errors.Errorf("id %s twice in one call", id)
		}
		seen[id] = struct{}{}
		if hidden[i] {
			hid[i] = 1
		}
		for _, cat := range categories[i] {
			cid, ok := c.catID[cat]
			if !ok {
				cid = int32(len(c.catName))
				c.catID[cat], c.catName = cid, append(c.catName, cat)
			}
			cats = append(cats, cid)
		}
		catOff[i+1] = int64(len(cats))
		replace[i] = -1
		if old, ok := c.slotOf[id]; ok {
			replace[i] = old
		}
	}
	slotOut := make([]int64, n)
	st := C.gorse_b200_vecdb_add_idf_vectors(c.handle, C.int64_t(n), i64p(aOff), i32p(aIDs), f32p(aIDF), C.int32_t(len(aIDF)), 0,
		i64p(bOff), i32p(bIDs), f32p(bIDF), C.int32_t(len(bIDF)), C.uint32_t(len(tagsIDF)), u8p(hid), C.int64_t(timestamp.UnixMilli()),
		i64p(catOff), i32p(cats), i64p(replace), i64p(slotOut))
	runtime.KeepAlive(aIDs)
	runtime.KeepAlive(bIDs)
	runtime.KeepAlive(aIDF)
	runtime.KeepAlive(bIDF)
	if err := b200Err(st); err != nil {
		return err
	}
	for i, id := range ids {
		if slotOut[i] < 0 {
			continue
		}
		c.slotOf[id] = slotOut[i]
		c.idOf = append(c.idOf, id)
		c.catsOf = append(c.catsOf, categories[i])
	}
	c.touch()
	return nil
}

// flattenCSR packs rows of ids as offsets [len(rows)+1] from 0 and the ids, as go/model/cf/b200.go does
func flattenCSR(rows [][]int32) ([]int64, []int32) {
	off := make([]int64, len(rows)+1)
	for r, row := range rows {
		off[r+1] = off[r] + int64(len(row))
	}
	idx := make([]int32, off[len(rows)])
	for r, row := range rows {
		copy(idx[off[r]:], row)
	}
	return off, idx
}

func (db *B200) GetVectors(ctx context.Context, name string, ids []string) ([]Vector, error) {
	if len(ids) == 0 {
		return []Vector{}, nil
	}
	if err := db.refresh(name); err != nil {
		return nil, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(name)
	if err != nil {
		return nil, err
	}
	found := make([]Vector, 0, len(ids))
	for _, id := range ids {
		slot, ok := c.slotOf[id]
		if !ok {
			continue
		}
		v, err := db.getSlot(c, slot)
		if err != nil {
			return nil, err
		}
		found = append(found, v)
	}
	return orderVectors(ids, found), nil // database.go:138-157
}

func (db *B200) getSlot(c *b200Collection, slot int64) (Vector, error) {
	v := Vector{Id: c.idOf[slot], Categories: c.catsOf[slot]}
	var hidden, live C.uint8_t
	var ts C.int64_t
	s := C.int64_t(slot)
	if c.info.Dimension > 0 {
		v.Values = make([]float32, c.info.Dimension)
		if err := b200Err(C.gorse_b200_vecdb_get(c.handle, &s, 1, f32p(v.Values), &hidden, &ts, &live)); err != nil {
			return v, err
		}
	} else {
		if err := b200Err(C.gorse_b200_vecdb_get(c.handle, &s, 1, nil, &hidden, &ts, &live)); err != nil {
			return v, err
		}
		var nnz C.int32_t
		if err := b200Err(C.gorse_b200_vecdb_get_sparse(c.handle, s, nil, nil, 0, &nnz)); err != nil {
			return v, err
		}
		v.Indices, v.Values = make([]uint32, nnz), make([]float32, nnz)
		if err := b200Err(C.gorse_b200_vecdb_get_sparse(c.handle, s, u32p(v.Indices), f32p(v.Values), nnz, &nnz)); err != nil {
			return v, err
		}
	}
	v.IsHidden, v.Timestamp = hidden != 0, time.UnixMilli(int64(ts)).UTC()
	return v, nil
}

func (db *B200) DeleteVectors(ctx context.Context, name string, timestamp time.Time) error {
	db.mu.Lock()
	defer db.mu.Unlock()
	c, err := db.collection(name)
	if err != nil {
		return err
	}
	slots := make([]int64, len(c.idOf))
	var count C.int64_t
	if err := b200Err(C.gorse_b200_vecdb_delete_before(c.handle, C.int64_t(timestamp.UnixMilli()), i64p(slots), C.int64_t(len(slots)), &count)); err != nil {
		return err
	}
	for _, slot := range slots[:count] {
		if c.slotOf[c.idOf[slot]] == slot {
			delete(c.slotOf, c.idOf[slot])
		}
	}
	if count > 0 {
		c.touch()
	}
	// the master rewrites every vector once per cycle and then deletes the old versions here: compacting once the dead
	// slots are as many as the live ones keeps a collection at most twice its live size
	var live, total C.int64_t
	if err := b200Err(C.gorse_b200_vecdb_count(c.handle, &live, &total)); err != nil {
		return err
	}
	if total-live >= live {
		if err := c.compact(); err != nil {
			return err
		}
	}
	// VectorWriter.Clean ends every rewrite here: the rewritten collection goes to disk now
	return db.save(name, c)
}

// QueryVectors: filter "hidden = false AND categories CONTAIN_ALL (...)" (xvec.go:381-389) evaluated on the device.
func (db *B200) QueryVectors(ctx context.Context, name string, q Vector, categories []string, topK int) ([]ScoredVector, error) {
	if topK <= 0 {
		return []ScoredVector{}, nil
	}
	if err := db.refresh(name); err != nil {
		return nil, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(name)
	if err != nil {
		return nil, err
	}
	want := make([]int32, 0, len(categories))
	for _, cat := range categories {
		id, ok := c.catID[cat]
		if !ok {
			return []ScoredVector{}, nil // nobody carries this category
		}
		want = append(want, id)
	}
	// no answer holds more than the live vectors: a large topK (the REST neighbour endpoints ask for
	// max(offset+n+|read items|, CacheSize)+1) allocates no more than the collection's size
	var live, total C.int64_t
	if err := b200Err(C.gorse_b200_vecdb_count(c.handle, &live, &total)); err != nil {
		return nil, err
	}
	if int64(topK) > int64(live) {
		topK = int(live)
	}
	if topK == 0 {
		return []ScoredVector{}, nil
	}
	slots, scores := make([]int64, topK), make([]float32, topK)
	var count C.int32_t
	var qOff []int64
	if c.info.Dimension == 0 {
		qOff = []int64{0, int64(len(q.Indices))}
	}
	st := C.gorse_b200_vecdb_query(c.handle, 1, f32p(q.Values), i64p(qOff), u32p(q.Indices), i32p(want), C.int32_t(len(want)),
		C.int32_t(topK), i64p(slots), f32p(scores), &count)
	if err := b200Err(st); err != nil {
		return nil, err
	}
	results := make([]ScoredVector, 0, count)
	for i := 0; i < int(count); i++ {
		v, err := db.getSlot(c, slots[i])
		if err != nil {
			return nil, err
		}
		results = append(results, ScoredVector{Vector: v, Score: scores[i]})
	}
	return results, nil
}

// QueryVectorsExcluding answers the worker's CF recall (worker/pipeline.go:403-449) for many users in one call: row i is
// QueryVectors(queries[i], nil, n+len(exclude[i])) without the ids in exclude[i] (the user's excludeSet,
// logics/recommend.go:67-80), so a row may hold more than n results, as in the reference.  The ids of one row must be distinct,
// as a set's are; ids the collection does not hold are passed as -1 and still count in topK.
func (db *B200) QueryVectorsExcluding(ctx context.Context, name string, queries [][]float32, exclude [][]string, n int) ([][]ScoredVector, error) {
	if len(queries) != len(exclude) {
		return nil, errors.Errorf("%d queries with %d exclude sets", len(queries), len(exclude))
	}
	results := make([][]ScoredVector, len(queries))
	if len(queries) == 0 || n <= 0 {
		return results, nil
	}
	if err := db.refresh(name); err != nil {
		return nil, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(name)
	if err != nil {
		return nil, err
	}
	dim := c.info.Dimension
	values := make([]float32, 0, len(queries)*dim)
	exOff := make([]int64, len(queries)+1)
	exSlots := []int64{}
	for i, q := range queries {
		if len(q) != dim {
			return nil, errors.Errorf("query %d has dimension %d, want %d", i, len(q), dim)
		}
		values = append(values, q...)
		for _, id := range exclude[i] {
			slot, ok := c.slotOf[id]
			if !ok {
				slot = -1
			}
			exSlots = append(exSlots, slot)
		}
		exOff[i+1] = int64(len(exSlots))
	}
	total := len(queries)*n + len(exSlots)
	slots, scores, counts := make([]int64, total), make([]float32, total), make([]int32, len(queries))
	var exact C.int64_t
	st := C.gorse_b200_vecdb_query_excluding(c.handle, C.int64_t(len(queries)), f32p(values), nil, 0, C.int32_t(n), i64p(exOff),
		i64p(exSlots), i64p(slots), f32p(scores), i32p(counts), &exact)
	runtime.KeepAlive(values)
	runtime.KeepAlive(exSlots)
	if err := b200Err(st); err != nil {
		return nil, err
	}
	log.Logger().Debug("batched CF recall", zap.Int("users", len(queries)), zap.Int64("exact_rows", int64(exact)))
	for i := range queries {
		start := int64(i)*int64(n) + exOff[i]
		row := make([]ScoredVector, 0, counts[i])
		for j := int64(0); j < int64(counts[i]); j++ {
			v, err := db.getSlot(c, slots[start+j])
			if err != nil {
				return nil, err
			}
			row = append(row, ScoredVector{Vector: v, Score: scores[start+j]})
		}
		results[i] = row
	}
	return results, nil
}

// ItemToItemRecommend answers the worker's item-to-item recommender (Recommender.recommendItemToItem,
// logics/recommend.go:244-283) for many users in one call on the collection ItemToItemCollection(name): row i is what the loop
// returns for a user with positive feedback contextIds[i] (in the order the loop visits them, newest first) and exclude set
// excludeIds[i] -- the neighbours of every context item (QueryItemToItem, logics/item_to_item.go:50-86) summed per id in
// float64 in context order, without the excluded ids, the best n.  scoreScale is 0.5 for type "auto", else 1.  Ids without a
// vector are passed as -1 (skipped as context, harmless as exclusions); the ids of one exclude set must be distinct, as a
// set's are.  Exact score ties are ordered by slot; the reference's map order there is unpinned.
func (db *B200) ItemToItemRecommend(ctx context.Context, collection string, contextIds [][]string, excludeIds [][]string, categories []string,
	n int, scoreScale float64) ([][]cache.Score, error) {
	if len(contextIds) != len(excludeIds) {
		return nil, errors.Errorf("%d context lists with %d exclude sets", len(contextIds), len(excludeIds))
	}
	results := make([][]cache.Score, len(contextIds))
	if len(contextIds) == 0 || n <= 0 {
		return results, nil
	}
	if err := db.refresh(collection); err != nil {
		return nil, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(collection)
	if err != nil {
		return nil, err
	}
	want := make([]int32, 0, len(categories))
	for _, cat := range categories {
		id, ok := c.catID[cat]
		if !ok {
			return results, nil // nobody carries this category: every neighbour list is empty
		}
		want = append(want, id)
	}
	slotsOf := func(lists [][]string) ([]int64, []int64) {
		off := make([]int64, len(lists)+1)
		slots := []int64{}
		for i, ids := range lists {
			for _, id := range ids {
				slot, ok := c.slotOf[id]
				if !ok {
					slot = -1
				}
				slots = append(slots, slot)
			}
			off[i+1] = int64(len(slots))
		}
		return off, slots
	}
	ctxOff, ctxSlots := slotsOf(contextIds)
	exOff, exSlots := slotsOf(excludeIds)
	users := len(contextIds)
	slots, scores, counts := make([]int64, users*n), make([]float64, users*n), make([]int32, users)
	stats := make([]int64, 4)
	st := C.gorse_b200_vecdb_item_to_item(c.handle, C.int64_t(users), i64p(ctxOff), i64p(ctxSlots), i64p(exOff), i64p(exSlots), i32p(want),
		C.int32_t(len(want)), C.int32_t(n), C.double(scoreScale), i64p(slots), (*C.double)(unsafe.Pointer(&scores[0])), i32p(counts), i64p(stats))
	runtime.KeepAlive(ctxSlots)
	runtime.KeepAlive(exSlots)
	runtime.KeepAlive(want)
	if err := b200Err(st); err != nil {
		return nil, err
	}
	log.Logger().Debug("batched item-to-item", zap.Int("users", users), zap.Int64("context_items", stats[0]), zap.Int64("exact_rows", stats[1]))
	for i := range results {
		row := make([]cache.Score, 0, counts[i])
		for j := i * n; j < i*n+int(counts[i]); j++ {
			row = append(row, cache.Score{Id: c.idOf[slots[j]], Score: scores[j], Categories: c.catsOf[slots[j]]})
		}
		results[i] = row
	}
	return results, nil
}

// UserToUserRecommend answers the worker's user-to-user recommender (Recommender.recommendUserToUser,
// logics/recommend.go:285-348) for many users in one call on the collection UserToUserCollection(name): row i is what the
// recommender returns for user userIds[i] with exclude set excludeIds[i] -- the first n similar users (QueryUserToUser,
// logics/user_to_user.go:50-86), each one's score added to every item of its positive feedback in float64 without the
// excluded ids, the best n, and of those only the items with itemOK set.  itemIds is the caller's item dictionary;
// feedback[userId] holds that user's positive feedback as indices into it (an item may repeat, once per positive feedback
// type); itemOK[j] reports whether itemIds[j] exists, is not hidden, is within ItemTTL and holds the requested categories.
// scoreScale is 0.5 for type "auto", else 1.  Users without a vector get an empty row; excluded ids outside the dictionary
// are harmless; the ids of one exclude set must be distinct, as a set's are.  Exact score ties are ordered by item index;
// the reference's map order there is unpinned.  The caller adds each item's categories from its own item metadata.
func (db *B200) UserToUserRecommend(ctx context.Context, collection string, userIds []string, itemIds []string, feedback map[string][]int32,
	itemOK []bool, excludeIds [][]string, n int, scoreScale float64) ([][]cache.Score, error) {
	if len(userIds) != len(excludeIds) {
		return nil, errors.Errorf("%d users with %d exclude sets", len(userIds), len(excludeIds))
	}
	if len(itemOK) != len(itemIds) {
		return nil, errors.Errorf("%d item flags for %d items", len(itemOK), len(itemIds))
	}
	results := make([][]cache.Score, len(userIds))
	if len(userIds) == 0 || n <= 0 {
		return results, nil
	}
	if err := db.refresh(collection); err != nil {
		return nil, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(collection)
	if err != nil {
		return nil, err
	}
	userSlots := make([]int64, len(userIds))
	for i, id := range userIds {
		slot, ok := c.slotOf[id]
		if !ok {
			slot = -1
		}
		userSlots[i] = slot
	}
	// the feedback rows by slot: only live slots can be neighbours
	rows := make([][]int32, len(c.idOf))
	for id, items := range feedback {
		if slot, ok := c.slotOf[id]; ok {
			rows[slot] = items
		}
	}
	fbOff := make([]int64, len(rows)+1)
	fbItems := []int32{}
	for s, items := range rows {
		for _, j := range items {
			if j < 0 || int(j) >= len(itemIds) {
				return nil, errors.Errorf("feedback of %s: item index %d outside the %d items", c.idOf[s], j, len(itemIds))
			}
		}
		fbItems = append(fbItems, items...)
		fbOff[s+1] = int64(len(fbItems))
	}
	okFlags := make([]uint8, len(itemIds))
	for j, v := range itemOK {
		if v {
			okFlags[j] = 1
		}
	}
	index := make(map[string]int64, len(itemIds))
	for j, id := range itemIds {
		index[id] = int64(j)
	}
	exOff := make([]int64, len(excludeIds)+1)
	exItems := []int64{}
	for i, ids := range excludeIds {
		for _, id := range ids {
			j, found := index[id]
			if !found {
				j = -1
			}
			exItems = append(exItems, j)
		}
		exOff[i+1] = int64(len(exItems))
	}
	users := len(userIds)
	items, scores, counts := make([]int64, users*n), make([]float64, users*n), make([]int32, users)
	stats := make([]int64, 4)
	st := C.gorse_b200_vecdb_user_to_user(c.handle, C.int64_t(users), i64p(userSlots), C.int64_t(len(rows)), i64p(fbOff), i32p(fbItems),
		C.int32_t(len(itemIds)), u8p(okFlags), i64p(exOff), i64p(exItems), C.int32_t(n), C.double(scoreScale), i64p(items),
		(*C.double)(unsafe.Pointer(&scores[0])), i32p(counts), i64p(stats))
	runtime.KeepAlive(userSlots)
	runtime.KeepAlive(fbItems)
	runtime.KeepAlive(okFlags)
	runtime.KeepAlive(exItems)
	if err := b200Err(st); err != nil {
		return nil, err
	}
	log.Logger().Debug("batched user-to-user", zap.Int("users", users), zap.Int64("query_users", stats[0]), zap.Int64("exact_rows", stats[1]))
	for i := range results {
		row := make([]cache.Score, 0, counts[i])
		for j := i * n; j < i*n+int(counts[i]); j++ {
			row = append(row, cache.Score{Id: itemIds[items[j]], Score: scores[j]})
		}
		results[i] = row
	}
	return results, nil
}

// NeighbourCache keeps the first n neighbours of the collection's vectors on the device between the item-to-item, session
// and user-to-user calls that ask for n neighbours without a category filter (gorse_b200_vecdb_neighbour_cache); every
// answer stays the same.  The pool holds min(live vectors, neighbour_cache_mb MB / (8 n + 4)) rows; the per-call work
// buffers of a cached call (the rows it computes and each table row's source, about 8 n + 12 bytes per row of the call)
// come on top of that budget.  The cache empties itself when the collection changes.  A reload replaces the collection's
// handle, which starts without a cache, so callers call this before each batch or request: with the same n and size it
// keeps what it holds and does nothing else.  With neighbour_cache_mb = 0, or an n outside [1, 1024] (which the
// neighbour entries themselves refuse or skip), it does nothing and returns nil.  An error wrapping
// storage.ErrNotSupported is a collection the cache does not serve (Cosine, or a sparse one with n above 128).  Answers do
// not depend on the cache, so a caller may go on without it after any error.
func (db *B200) NeighbourCache(name string, n int) error {
	if db.cacheMB == 0 || n < 1 || n > 1024 {
		return nil
	}
	if err := db.refresh(name); err != nil {
		return err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(name)
	if err != nil {
		return err
	}
	if err := db.sizeNeighbourCache(c, n); err != nil {
		return err
	}
	c.nbrOnce.Do(func() { db.loadNeighbours(name, c, n) })
	return nil
}

// sizeNeighbourCache turns on c's neighbour cache at n with min(live vectors, neighbour_cache_mb MB / (8 n + 4)) rows; the
// same n and size again keep what it holds
func (db *B200) sizeNeighbourCache(c *b200Collection, n int) error {
	rows := min(int64(len(c.slotOf)), (db.cacheMB<<20)/(8*int64(n)+4))
	st := C.gorse_b200_vecdb_neighbour_cache(c.handle, C.int32_t(n), C.int64_t(rows))
	if st == C.GORSE_B200_ERR_UNSUPPORTED { // a Cosine collection, or n above 128 for a sparse one
		return fmt.Errorf("%s: %w", C.GoString(C.gorse_b200_last_error()), storage.ErrNotSupported)
	}
	return b200Err(st)
}

// SessionRecommend answers the REST server's session recommendation (RestServer.sessionRecommend, server/rest.go:1069-1173)
// for many sessions in one call on the collection ItemToItemCollection(name) of the first item-to-item recommender: row i
// is the TopKFilter(top) of the handler for a session whose positive feedback items are contextIds[i] (in the order the
// handler visits them, after data.SortFeedbacks and the positive feedback types) and whose items, of every feedback type,
// are excludeIds[i].  Each context item's neighbours are QueryItemToItem(item, nil, n) (logics/item_to_item.go:50-86);
// only the ones itemOK passes are kept; an item whose kept list is not empty counts, and the walk stops at the
// contextSize-th one; the kept neighbours not in the exclude set are summed per id in float64 in context order.  top is
// n + offset of the request; the caller slices [offset:].  scoreScale is 0.5 for type "auto", else 1.
//
// itemOK is FilterVisibleItemsByCategories (rest.go:815-832) for the request's categories: it receives the collection's
// live ids once per call and returns, per id, whether the item exists in the data store, is not hidden and holds every
// requested category; nil passes every id.  Every session of one call shares it, so a caller batches requests by
// category.  Ids without a vector are passed as -1 (they give an empty list and do not count); the ids of one exclude set
// must be distinct, as a set's are.  Exact score ties are ordered by slot; the reference's map order there is unpinned.
// An error wrapping storage.ErrNotSupported (top above 1024, n outside the collection's limits, a Cosine collection) means
// the caller runs the handler's own loop.
func (db *B200) SessionRecommend(ctx context.Context, collection string, contextIds [][]string, excludeIds [][]string,
	itemOK func(ids []string) ([]bool, error), n, contextSize, top int, scoreScale float64) ([][]cache.Score, error) {
	if len(contextIds) != len(excludeIds) {
		return nil, errors.Errorf("%d context lists with %d exclude sets", len(contextIds), len(excludeIds))
	}
	results := make([][]cache.Score, len(contextIds))
	if len(contextIds) == 0 || top <= 0 {
		return results, nil
	}
	if err := db.refresh(collection); err != nil {
		return nil, err
	}
	db.mu.RLock()
	defer db.mu.RUnlock()
	c, err := db.collection(collection)
	if err != nil {
		return nil, err
	}
	var okFlags []uint8
	if itemOK != nil {
		// one flag per slot: the live ids are asked once, dead slots (never neighbours) stay 0
		slots := make([]int64, 0, len(c.slotOf))
		ids := make([]string, 0, len(c.slotOf))
		for id, slot := range c.slotOf {
			ids = append(ids, id)
			slots = append(slots, slot)
		}
		flags, err := itemOK(ids)
		if err != nil {
			return nil, err
		}
		if len(flags) != len(ids) {
			return nil, errors.Errorf("%d item flags for %d ids", len(flags), len(ids))
		}
		okFlags = make([]uint8, max(len(c.idOf), 1))
		for i, v := range flags {
			if v {
				okFlags[slots[i]] = 1
			}
		}
	}
	slotsOf := func(lists [][]string) ([]int64, []int64) {
		off := make([]int64, len(lists)+1)
		slots := []int64{}
		for i, ids := range lists {
			for _, id := range ids {
				slot, ok := c.slotOf[id]
				if !ok {
					slot = -1
				}
				slots = append(slots, slot)
			}
			off[i+1] = int64(len(slots))
		}
		return off, slots
	}
	ctxOff, ctxSlots := slotsOf(contextIds)
	exOff, exSlots := slotsOf(excludeIds)
	sessions := len(contextIds)
	slots, scores, counts := make([]int64, sessions*top), make([]float64, sessions*top), make([]int32, sessions)
	stats := make([]int64, 4)
	st := C.gorse_b200_vecdb_session_recommend(c.handle, C.int64_t(sessions), i64p(ctxOff), i64p(ctxSlots), i64p(exOff), i64p(exSlots),
		u8p(okFlags), C.int32_t(n), C.int32_t(contextSize), C.int32_t(top), C.double(scoreScale), i64p(slots),
		(*C.double)(unsafe.Pointer(&scores[0])), i32p(counts), i64p(stats))
	runtime.KeepAlive(ctxSlots)
	runtime.KeepAlive(exSlots)
	runtime.KeepAlive(okFlags)
	if st == C.GORSE_B200_ERR_UNSUPPORTED {
		return nil, fmt.Errorf("%s: %w", C.GoString(C.gorse_b200_last_error()), storage.ErrNotSupported)
	}
	if err := b200Err(st); err != nil {
		return nil, err
	}
	log.Logger().Debug("batched session recommendation", zap.Int("sessions", sessions), zap.Int64("context_items", stats[0]),
		zap.Int64("exact_rows", stats[1]))
	for i := range results {
		row := make([]cache.Score, 0, counts[i])
		for j := i * top; j < i*top+int(counts[i]); j++ {
			row = append(row, cache.Score{Id: c.idOf[slots[j]], Score: scores[j], Categories: c.catsOf[slots[j]]})
		}
		results[i] = row
	}
	return results, nil
}

func f32p(s []float32) *C.float {
	if len(s) == 0 {
		return nil
	}
	return (*C.float)(unsafe.Pointer(&s[0]))
}
func i64p(s []int64) *C.int64_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int64_t)(unsafe.Pointer(&s[0]))
}
func i32p(s []int32) *C.int32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int32_t)(unsafe.Pointer(&s[0]))
}
func u32p(s []uint32) *C.uint32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint32_t)(unsafe.Pointer(&s[0]))
}
func u8p(s []uint8) *C.uint8_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&s[0]))
}

// ---- collections on disk (a root in the URL) ----
//
// File <root>/<tablePrefix><name>.b200vec: the shim's header, little-endian --
//   magic "GB200SHM", u32 version 1, i64 generation (the writer's clock in ns at the save), i32 dimension, i32 distance,
//   u32 category names then each as u32 length + bytes, u64 vectors then per vector in saved-slot order its id (u32 length +
//   bytes) and its categories (u32 count + u32 name indices)
// -- then the library's stream (gorse_b200_vecdb_save; format in include/gorse_b200.h), whose vector i is the header's i-th.
// A save writes <file>.tmp, fsyncs it and renames it into place, so a reader sees the previous file until the rename.

const b200FileSuffix = ".b200vec"

var b200FileMagic = [8]byte{'G', 'B', '2', '0', '0', 'S', 'H', 'M'}

func (db *B200) path(name string) string {
	return filepath.Join(db.root, db.tablePrefix+name+b200FileSuffix)
}

// touch marks a write of this process: the collection is saved by the next save point or 5 s after its last write
func (c *b200Collection) touch() {
	c.dirty, c.lastWrite = true, time.Now()
}

// flush saves every collection that has seen no write for 5 s: the CF hand-off (master/tasks.go:930-961) ends without a
// closing call
func (db *B200) flush() {
	defer db.flusher.Done()
	tick := time.NewTicker(time.Second)
	defer tick.Stop()
	for {
		select {
		case <-db.stop:
			return
		case <-tick.C:
		}
		db.mu.Lock()
		for name, c := range db.collections {
			if c.dirty && time.Since(c.lastWrite) >= 5*time.Second {
				if err := db.save(name, c); err != nil {
					log.Logger().Error("save vector collection", zap.String("collection", name), zap.Error(err))
				}
			}
		}
		db.mu.Unlock()
	}
}

// save writes a collection with unsaved writes to its file; the caller holds db.mu for writing
func (db *B200) save(name string, c *b200Collection) error {
	if db.root == "" || !c.dirty {
		return nil
	}
	path := db.path(name)
	f, err := os.Create(path + ".tmp")
	if err != nil {
		return errors.Trace(err)
	}
	defer os.Remove(path + ".tmp") // after a successful rename there is nothing to remove
	generation := time.Now().UnixNano()
	if generation <= c.generation {
		generation = c.generation + 1
	}
	// the library's live slots are the stream's vectors (an id added twice in one call holds two live slots)
	slots, live := make([]int64, len(c.idOf)), make([]uint8, len(c.idOf))
	for i := range slots {
		slots[i] = int64(i)
	}
	if err := b200Err(C.gorse_b200_vecdb_get(c.handle, i64p(slots), C.int64_t(len(slots)), nil, nil, nil, u8p(live))); err != nil {
		f.Close()
		return err
	}
	w := bufio.NewWriterSize(f, 1<<20)
	if err := c.writeHeader(w, generation, live); err != nil {
		f.Close()
		return err
	}
	h := cgo.NewHandle(io.Writer(w))
	st := C.gorse_b200_vecdb_save(c.handle, C.gorse_b200_snapshot_write_ptr(), unsafe.Pointer(&h), nil, nil)
	h.Delete()
	if err := b200Err(st); err != nil {
		f.Close()
		return err
	}
	if err := w.Flush(); err != nil {
		f.Close()
		return errors.Trace(err)
	}
	if err := f.Sync(); err != nil {
		f.Close()
		return errors.Trace(err)
	}
	if err := f.Close(); err != nil {
		return errors.Trace(err)
	}
	// the lists of this generation are in place before the collection file is: a reader that reloads the new file finds
	// them at once
	db.saveNeighbours(name, c, generation)
	if err := os.Rename(path+".tmp", path); err != nil {
		return errors.Trace(err)
	}
	st2, err := os.Stat(path)
	if err != nil {
		return errors.Trace(err)
	}
	c.generation, c.file, c.dirty = generation, st2, false
	return nil
}

// ---- neighbour lists on disk (neighbour_fill_n in the URL) ----
//
// File <root>/<tablePrefix><name>.b200vec.nbr: magic "GB200NBS", u32 version 1, i64 generation (the collection file's),
// i32 n, then the library's neighbour stream (gorse_b200_vecdb_neighbour_cache_save; format in include/gorse_b200.h).  The
// process that writes an item-to-item or user-to-user collection fills its neighbour cache at neighbour_fill_n and renames
// this file into place before the collection file of the same generation, so a reader that loads the new collection file
// finds the lists already there; every process that loads the collection loads the lists when the generation matches, so
// its first batches and sessions start warm.  The library refuses lists of another collection itself (their
// fingerprint).  Lists only save work: every failure is logged and the process goes on cold.

const b200NbrSuffix = ".nbr"

var b200NbrMagic = [8]byte{'G', 'B', '2', '0', '0', 'N', 'B', 'S'}

func b200FillsNeighbours(name string) bool {
	return strings.HasPrefix(name, ItemToItemPrefix+"_") || strings.HasPrefix(name, UserToUserPrefix+"_")
}

// saveNeighbours fills c's neighbour cache at neighbour_fill_n and writes <file>.nbr (tmp, fsync, rename) with the
// generation of the collection file being saved; the caller holds db.mu for writing and renames the collection file into
// place afterwards.  A process whose cache was off (the master, which never reads the lists) turns it off again, so the
// pool does not stay on its device.
func (db *B200) saveNeighbours(name string, c *b200Collection, generation int64) {
	if db.fillN == 0 || db.cacheMB == 0 || !b200FillsNeighbours(name) {
		return
	}
	stats := make([]int64, 7)
	if err := b200Err(C.gorse_b200_vecdb_neighbour_cache_stats(c.handle, i64p(stats))); err != nil {
		log.Logger().Warn("save neighbour lists; readers start cold", zap.String("collection", name), zap.Error(err))
		return
	}
	if err := db.writeNeighbours(name, c, generation); err != nil {
		log.Logger().Warn("save neighbour lists; readers start cold", zap.String("collection", name), zap.Error(err))
	}
	if stats[1] == 0 { // the capacity before the fill: off
		if err := b200Err(C.gorse_b200_vecdb_neighbour_cache(c.handle, C.int32_t(db.fillN), 0)); err != nil {
			log.Logger().Warn("turn the neighbour cache off after saving it", zap.String("collection", name), zap.Error(err))
		}
	}
}

func (db *B200) writeNeighbours(name string, c *b200Collection, generation int64) error {
	if err := db.sizeNeighbourCache(c, db.fillN); err != nil {
		return err
	}
	if err := b200Err(C.gorse_b200_vecdb_neighbour_cache_fill(c.handle, nil)); err != nil {
		return err
	}
	path := db.path(name) + b200NbrSuffix
	f, err := os.Create(path + ".tmp")
	if err != nil {
		return errors.Trace(err)
	}
	defer os.Remove(path + ".tmp")
	le := binary.LittleEndian
	head := le.AppendUint32(append([]byte{}, b200NbrMagic[:]...), 1)
	head = le.AppendUint64(head, uint64(generation))
	head = le.AppendUint32(head, uint32(int32(db.fillN)))
	w := bufio.NewWriterSize(f, 1<<20)
	if _, err := w.Write(head); err != nil {
		f.Close()
		return errors.Trace(err)
	}
	h := cgo.NewHandle(io.Writer(w))
	st := C.gorse_b200_vecdb_neighbour_cache_save(c.handle, C.gorse_b200_snapshot_write_ptr(), unsafe.Pointer(&h), nil)
	h.Delete()
	if err := b200Err(st); err != nil {
		f.Close()
		return err
	}
	if err := w.Flush(); err != nil {
		f.Close()
		return errors.Trace(err)
	}
	if err := f.Sync(); err != nil {
		f.Close()
		return errors.Trace(err)
	}
	if err := f.Close(); err != nil {
		return errors.Trace(err)
	}
	return errors.Trace(os.Rename(path+".tmp", path))
}

// loadNeighbours loads <file>.nbr into c's neighbour cache when it carries c's generation and, with n > 0, lists of n
// neighbours (n = 0: the file's n).  A missing file, another generation or n, and every failure leave c cold.
func (db *B200) loadNeighbours(name string, c *b200Collection, n int) {
	if db.root == "" || db.cacheMB == 0 || !b200FillsNeighbours(name) {
		return
	}
	warn := func(err error) {
		log.Logger().Warn("load neighbour lists; going on cold", zap.String("collection", name), zap.Error(err))
	}
	f, err := os.Open(db.path(name) + b200NbrSuffix)
	if err != nil {
		if !os.IsNotExist(err) {
			warn(errors.Trace(err))
		}
		return
	}
	defer f.Close()
	le := binary.LittleEndian
	r := bufio.NewReaderSize(f, 1<<20)
	var head [24]byte
	if _, err := io.ReadFull(r, head[:]); err != nil || [8]byte(head[:8]) != b200NbrMagic || le.Uint32(head[8:]) != 1 {
		warn(errors.New("not a b200 neighbour file of version 1"))
		return
	}
	fileN := int(int32(le.Uint32(head[20:])))
	if int64(le.Uint64(head[12:])) != c.generation || (n > 0 && fileN != n) {
		return // lists of another save, or of another n: this process computes its own
	}
	if err := db.sizeNeighbourCache(c, fileN); err != nil {
		warn(err)
		return
	}
	h := cgo.NewHandle(io.Reader(r))
	st := C.gorse_b200_vecdb_neighbour_cache_load(c.handle, C.gorse_b200_snapshot_read_ptr(), unsafe.Pointer(&h), nil)
	h.Delete()
	if err := b200Err(st); err != nil {
		warn(err)
	}
}

// writeHeader writes the shim's header: the ids of the live slots in slot order, which is the order of the library's stream
func (c *b200Collection) writeHeader(w io.Writer, generation int64, live []uint8) error {
	le := binary.LittleEndian
	buf := append([]byte{}, b200FileMagic[:]...)
	buf = le.AppendUint32(buf, 1)
	buf = le.AppendUint64(buf, uint64(generation))
	buf = le.AppendUint32(buf, uint32(int32(c.info.Dimension)))
	buf = le.AppendUint32(buf, uint32(int32(c.info.Distance)))
	buf = le.AppendUint32(buf, uint32(len(c.catName)))
	for _, s := range c.catName {
		buf = le.AppendUint32(buf, uint32(len(s)))
		buf = append(buf, s...)
	}
	n := 0
	for _, l := range live {
		n += int(l)
	}
	buf = le.AppendUint64(buf, uint64(n))
	for slot, id := range c.idOf {
		if live[slot] == 0 {
			continue // a deleted slot: not in the stream
		}
		buf = le.AppendUint32(buf, uint32(len(id)))
		buf = append(buf, id...)
		buf = le.AppendUint32(buf, uint32(len(c.catsOf[slot])))
		for _, cat := range c.catsOf[slot] {
			buf = le.AppendUint32(buf, uint32(c.catID[cat]))
		}
	}
	_, err := w.Write(buf)
	return errors.Trace(err)
}

// refresh reloads a collection whose file another process has replaced since this one last saved or loaded it, and forgets
// one whose file another process has removed (DeleteCollection on the master: the CF collection of an older model); slot
// maps taken earlier go stale, as after a compaction
func (db *B200) refresh(name string) error {
	if db.root == "" {
		return nil
	}
	st, err := os.Stat(db.path(name))
	if os.IsNotExist(err) {
		db.mu.Lock()
		defer db.mu.Unlock()
		if c, ok := db.collections[name]; ok && !c.dirty && c.generation > 0 {
			delete(db.collections, name)
			return b200Err(C.gorse_b200_vecdb_destroy(c.handle))
		}
		return nil // never saved, or writes not saved yet: what this process holds stands
	}
	if err != nil {
		return errors.Trace(err)
	}
	db.mu.RLock()
	c, ok := db.collections[name]
	current := ok && (c.dirty || sameFile(st, c.file))
	db.mu.RUnlock()
	if current {
		return nil
	}
	db.mu.Lock()
	defer db.mu.Unlock()
	return db.reload(name)
}

// sameFile: the file last saved or loaded is still in place.  Every save renames a new file into place, so the inode
// changes even when two saves land in one tick of a coarse modification time.
func sameFile(st, last os.FileInfo) bool {
	return last != nil && os.SameFile(st, last) && st.Size() == last.Size() && st.ModTime().Equal(last.ModTime())
}

// reload loads <root>/<name> when its generation is newer than the collection this process holds (or it holds none) and
// swaps the handle and the id maps; the caller holds db.mu for writing
func (db *B200) reload(name string) error {
	old, ok := db.collections[name]
	if ok && old.dirty {
		return nil
	}
	f, err := os.Open(db.path(name))
	if err != nil {
		return errors.Trace(err)
	}
	defer f.Close()
	st, err := f.Stat()
	if err != nil {
		return errors.Trace(err)
	}
	r := bufio.NewReaderSize(f, 1<<20)
	c, err := readHeader(r, name)
	if err != nil {
		return errors.Annotatef(err, "vector collection file %s", db.path(name))
	}
	c.file = st
	if ok && c.generation <= old.generation {
		old.file = st
		return nil
	}
	h := cgo.NewHandle(io.Reader(r))
	var count C.int64_t
	status := C.gorse_b200_vecdb_load(db.ctx, C.gorse_b200_snapshot_read_ptr(), unsafe.Pointer(&h), &c.handle, nil)
	h.Delete()
	if err := b200Err(status); err != nil {
		return errors.Annotatef(err, "vector collection file %s", db.path(name))
	}
	if err := b200Err(C.gorse_b200_vecdb_count(c.handle, &count, nil)); err != nil || int(count) != len(c.idOf) {
		C.gorse_b200_vecdb_destroy(c.handle)
		return errors.Errorf("vector collection file %s: %d ids for %d vectors", db.path(name), len(c.idOf), int64(count))
	}
	if ok {
		C.gorse_b200_vecdb_destroy(old.handle)
	}
	db.collections[name] = c
	c.nbrOnce.Do(func() { db.loadNeighbours(name, c, 0) })
	return nil
}

// readHeader reads the shim's header into a collection without a handle
func readHeader(r io.Reader, name string) (*b200Collection, error) {
	le := binary.LittleEndian
	var fixed [32]byte
	if _, err := io.ReadFull(r, fixed[:]); err != nil {
		return nil, errors.Trace(err)
	}
	if [8]byte(fixed[:8]) != b200FileMagic || le.Uint32(fixed[8:]) != 1 {
		return nil, errors.New("not a b200 collection file of version 1")
	}
	c := &b200Collection{info: CollectionInfo{Name: name, Dimension: int(int32(le.Uint32(fixed[20:]))), Distance: Distance(int32(le.Uint32(fixed[24:])))},
		slotOf: map[string]int64{}, catID: map[string]int32{}, generation: int64(le.Uint64(fixed[12:]))}
	u32 := func() (uint32, error) {
		var b [4]byte
		_, err := io.ReadFull(r, b[:])
		return le.Uint32(b[:]), err
	}
	str := func() (string, error) {
		n, err := u32()
		if err != nil {
			return "", err
		}
		b := make([]byte, n)
		_, err = io.ReadFull(r, b)
		return string(b), err
	}
	nCats := le.Uint32(fixed[28:])
	for i := uint32(0); i < nCats; i++ {
		s, err := str()
		if err != nil {
			return nil, errors.Trace(err)
		}
		c.catID[s], c.catName = int32(i), append(c.catName, s)
	}
	var nb [8]byte
	if _, err := io.ReadFull(r, nb[:]); err != nil {
		return nil, errors.Trace(err)
	}
	n := le.Uint64(nb[:])
	for slot := uint64(0); slot < n; slot++ {
		id, err := str()
		if err != nil {
			return nil, errors.Trace(err)
		}
		k, err := u32()
		if err != nil {
			return nil, errors.Trace(err)
		}
		cats := make([]string, 0, k)
		for j := uint32(0); j < k; j++ {
			x, err := u32()
			if err != nil {
				return nil, errors.Trace(err)
			}
			if x >= nCats {
				return nil, errors.Errorf("category %d of %d names", x, nCats)
			}
			cats = append(cats, c.catName[x])
		}
		c.slotOf[id] = int64(slot) // an id held twice: the later slot, as after the add
		c.idOf, c.catsOf = append(c.idOf, id), append(c.catsOf, cats)
	}
	return c, nil
}

//export gorseB200SnapshotWrite
func gorseB200SnapshotWrite(user unsafe.Pointer, buf unsafe.Pointer, n C.int64_t) C.int32_t {
	w := (*(*cgo.Handle)(user)).Value().(io.Writer) // user = &handle, the documented way to carry a Handle in a void*
	if _, err := w.Write(unsafe.Slice((*byte)(buf), int(n))); err != nil {
		return 1
	}
	return 0
}

//export gorseB200SnapshotRead
func gorseB200SnapshotRead(user unsafe.Pointer, buf unsafe.Pointer, n C.int64_t) C.int64_t {
	r := (*(*cgo.Handle)(user)).Value().(io.Reader)
	k, err := io.ReadAtLeast(r, unsafe.Slice((*byte)(buf), int(n)), 1)
	if k > 0 {
		return C.int64_t(k)
	}
	if err == io.EOF {
		return 0
	}
	return -1
}
