"""Device memory the library holds (gorse_b200_device_bytes): closing every handle and then the context gives back all they
allocated, a one-shot call gives back its scratch before it returns, and a call that fails after allocating leaves nothing
behind and raises the error it always raised."""
import io

import numpy as np
import pytest

import fm_oracle
from gorse_b200 import _lib, synth

pytestmark = pytest.mark.gpu

U, I, D = 300, 200, 32   # users, items, factors
NU = 20                  # users of the batched calls


def feedback():
    off, items = synth.make_feedback(U, I, 3000, seed=0)
    return off, items, synth.leave_one_out(off, items, seed=1)[1]


def id_rows(rng, n, width, hi):
    """n sorted lists of 1 .. width distinct ids below hi"""
    return [np.sort(rng.choice(hi, int(rng.integers(1, width + 1)), replace=False)) for _ in range(n)]


def sparse_vectors(rng, n):
    return [(ids.astype(np.uint32), rng.uniform(0.1, 1.0, ids.size).astype(np.float32)) for ids in id_rows(rng, n, 12, 400)]


def unchanged(gb, call):
    """call()'s result, after checking that the call left the library's device bytes as it found them"""
    before = gb.device_bytes()
    out = call()
    assert gb.device_bytes() == before
    return out


def exercise_collection(gb, col, q, fb_lists):
    """every read entry of a collection, each growing the collection's work buffers"""
    col.query(q, (), 10)
    ctx_lists = [[u % 50, (u * 7) % 50, -1] for u in range(NU)]
    col.item_to_item(ctx_lists, [[u % 50] for u in range(NU)], 5)
    col.session_recommend(ctx_lists, [[] for _ in range(NU)], 5, 2, 5)
    col.user_to_user(np.arange(NU), fb_lists, [[] for _ in range(NU)], 5, I)
    if col.dim > 0:
        col.query_excluding(q, [[0, 1] for _ in range(len(q))], 10)


def save_load_compact(gb, ctx, col, q):
    buf = io.BytesIO()
    col.save(buf)
    with gb.VectorCollection.load(ctx, io.BytesIO(buf.getvalue())) as loaded:
        loaded.query(q, (), 10)
    col.delete_before(30)
    col.compact()
    col.query(q, (), 10)


def test_closing_every_handle_returns_every_byte(gb):
    rng = np.random.default_rng(0)
    off, items, (toff, titems) = feedback()
    ioff, iusers = gb.transpose_csr(off, items, I)
    fb_lists = [items[off[u]:off[u + 1]] for u in range(U)]
    base = gb.device_bytes()
    with gb.Context(0) as ctx:
        with gb.CFModel(ctx, U, I, D, off, items, ioff, iusers) as m:
            m.init_normal(0.0, 0.1, 1)
            m.bpr_epoch(0.05, 0.01, int(off[-1]), 1)
            m.als_epoch(0.06, 0.001)
            m.fit("bpr", toff, titems, None, None, n_epochs=2, verbose=1, candidates=20)
            m.fit("als", toff, titems, None, None, n_epochs=2, verbose=1, candidates=20)
            m.fit_trials([("bpr", dict(lr=0.05, n_epochs=2, verbose=1, candidates=20)), ("als", dict(reg=0.06, n_epochs=2, verbose=1, candidates=20))],
                         toff, titems, None, None)
            with m.eval_plan(toff, titems, n_candidates=20) as plan:
                plan.run()
            P, Q = m.get_factors()
            assert gb.device_bytes() > base
        with gb.BruteforceIndex(ctx, D, gb.METRIC_NEG_DOT) as ix:
            ix.add(Q)
            ix.search_indices(np.arange(16), 10)
            ix.search_vectors(P[:16], 10)
        with gb.SparseIndex(ctx) as sx:
            vecs = sparse_vectors(rng, 500)
            sx.add(np.concatenate([[0], np.cumsum([v[0].size for v in vecs])]), np.concatenate([v[0] for v in vecs]),
                   np.concatenate([v[1] for v in vecs]))
            sx.search_range(0, 500, 10)
        nf, k = 500, 8
        with gb.VectorCollection(ctx, D, gb.DISTANCE_DOT) as item_col, gb.VectorCollection(ctx, D, gb.DISTANCE_EUCLIDEAN) as user_col, \
                gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as sparse_col, \
                gb.FMRanker(ctx, nf, k, 6, 1024, (), fm_oracle.random_params(rng, nf, k)) as fm:
            item_col.add(values=Q, timestamps=np.arange(I), categories=[[i % 3] for i in range(I)])
            user_col.add(values=P, timestamps=np.arange(U))
            sparse_col.add(sparse=sparse_vectors(rng, U), timestamps=np.arange(U))
            sparse_col.add_idf_vectors(id_rows(rng, 50, 8, 100), rng.uniform(0.5, 2.0, 100), timestamp_ms=U)
            fm.rank(fm_oracle.random_input(rng, nf, [10] * NU, I))
            exercise_collection(gb, item_col, P[:NU], fb_lists)
            exercise_collection(gb, sparse_col, sparse_vectors(rng, NU), fb_lists)
            stages = [gb.ListStage(np.arange(10, dtype=np.int32), np.linspace(1.0, 0.0, 10)), gb.CollaborativeStage(),
                      gb.ItemToItemStage(item_col, 5, [[u % I, (u + 3) % I] for u in range(NU)], np.arange(I), np.arange(I)),
                      gb.UserToUserStage(user_col, 5, np.arange(NU), fb_lists)]
            cf = (item_col, P[:NU], np.arange(I), np.arange(I), 10)
            gb.recommend(ctx, [[] for _ in range(NU)], I, np.ones(I, np.uint8), stages, cf=cf,
                         ranker=(fm, fm_oracle.random_input(rng, nf, [0] * NU, I)))
            save_load_compact(gb, ctx, item_col, P[:NU])
            save_load_compact(gb, ctx, sparse_col, sparse_vectors(rng, NU))
    assert gb.device_bytes() == base


def test_one_shot_calls_return_their_scratch(gb):
    rng = np.random.default_rng(1)
    off, items, (toff, titems) = feedback()
    nf, k, nd = 300, 8, 3
    train, test = fm_oracle.random_ctr(rng, nf, 500, n_ids=40), fm_oracle.random_ctr(rng, nf, 200, n_ids=40)
    p0 = fm_oracle.init_params(rng, nf, k)
    with gb.Context(0) as ctx, gb.CFModel(ctx, U, I, D, off, items) as m:
        m.init_normal(0.0, 0.1, 2)
        unchanged(gb, lambda: m.predict(rng.integers(0, U, 100), rng.integers(0, I, 100)))
        t = unchanged(gb, lambda: m.bpr_sample_triples(7, 0, 512))
        unchanged(gb, lambda: m.bpr_apply_triples(t, 0.05, 0.01, gb.SCATTER_STORE, gb.ORDER_SEQUENTIAL))
        unchanged(gb, lambda: m.bpr_apply_triples(t, 0.05, 0.01, gb.SCATTER_ATOMIC, gb.ORDER_HOGWILD))
        trainer = gb.FMTrainer(ctx, nf, nd, n_factors=k, n_epochs=2, verbose=1)
        unchanged(gb, lambda: trainer.fit(train, test, p0))
        unchanged(gb, lambda: trainer.fit_trials([{}, {"lr": 0.01}], train, test, [p0, p0]))
        unchanged(gb, lambda: gb.ranker_gauc(ctx, nf, k, nd, p0, test, 40, gb.user_feedback_counts(train, 40), context_size=4))
        emb = rng.standard_normal((I, 16)).astype(np.float32)
        unchanged(gb, lambda: gb.evaluate_embeddings(ctx, emb, None, (off, items), (toff, titems), (off, items), n_candidates=20))


def test_failures_after_allocation_leave_nothing(gb):
    rng = np.random.default_rng(2)
    with gb.Context(0) as ctx:
        with gb.VectorCollection(ctx, 64, gb.DISTANCE_DOT) as col:
            col.add(values=rng.standard_normal((500, 64)).astype(np.float32))
            buf = io.BytesIO()
            col.save(buf)
        cut = buf.getvalue()[:-4 * 64 * 10]   # ten rows short: the load has reserved the rows on the device by then
        before = gb.device_bytes()
        with pytest.raises(gb.GorseB200Error) as ei:
            gb.VectorCollection.load(ctx, io.BytesIO(cut))
        assert ei.value.status == _lib.ERR_ARG and f"ends at byte {len(cut)}, inside values" in ei.value.message
        assert gb.device_bytes() == before
        with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as sparse_col:
            idf = rng.uniform(0.5, 2.0, 100).astype(np.float32)
            sparse_col.add_idf_vectors(id_rows(rng, 50, 8, 100), idf, timestamp_ms=1)
            idf[3] = np.nan
            before = gb.device_bytes()
            with pytest.raises(gb.GorseB200Error) as ei:
                sparse_col.add_idf_vectors([[5, 4], [3, 9]], idf)
            assert ei.value.status == _lib.ERR_ARG and "NaN" in ei.value.message
            assert gb.device_bytes() == before
