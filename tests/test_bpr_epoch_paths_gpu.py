"""Every BPR epoch kernel against the oracle, on the rows that only one triple of the epoch touches.

`gorse_b200_bpr_epoch` picks its kernel from the scatter mode and d:

  scatter  d                      kernel
  ATOMIC   16, 32, 64, 128        bpr_round_kernel<C>: one cooperative launch, rounds of 8192 triples
  ATOMIC   other multiples of 16  bpr_round_delta_quad_kernel + bpr_round_add_kernel, two launches per round
  ATOMIC   d % 16 != 0            bpr_round_delta_any_kernel + bpr_round_add_kernel, two launches per round
  STORE    16, 32, 64, 128        bpr_epoch_kernel<C>, software-pipelined, free-running
  STORE    other multiples of 16  bpr_epoch_kernel<0>, two passes over the rows, free-running
  STORE    d % 16 != 0            bpr_epoch_any_kernel, one thread per triple, free-running

A store-scatter epoch is free-running by contract, so which update of a shared row wins depends on scheduling.  A live
triple (j >= 0) whose user, positive and negative no other live triple of the epoch touches is ISOLATED: its rows end
the epoch as one step from their initial values, whatever the schedule, and the oracle (the reference with Jobs = 1)
computes that step.  So the test draws the epoch's triple stream with bpr_sample_triples (the same counter RNG and
seed), applies the isolated triples with the oracle on a compact copy of their rows, and checks after the epoch:

  - isolated rows, STORE: bit-identical to the oracle;
  - isolated rows, ATOMIC: |got - want| <= 2 spacing(|before| + |want|) per element.  The device adds fl(lr t) to
    the row where the oracle may fuse lr t + row into one rounding, and |lr t| <= |before| + |want|;
  - rows no live triple touches: bit-identical to before;
  - every row: finite.

That bound is per element, so it sees an error in a small row that the round model's 1e-5 of the table's largest
factor (test_bpr_rounds_gpu.py) cannot.  Factors start at std 0.1, so that no expected value is subnormal
(red.global.add.f32 flushes subnormal results).

Sizing.  Items are uniform (zipf_s = 0) and every user has ~2 items; 1000 users without feedback are appended so that
the sampler goes through the list of active users.  With n steps over U users and I items, a user is touched by no
other triple with probability ~exp(-n/U) and an item with ~exp(-2n/I), so a triple is isolated with probability
~exp(-n/U - 4n/I).  At U = 1M, I = 2M, n = 450K that is exp(-1.35) ~ 0.26: ~115K isolated triples.  Every
grid-stride loop must run at least 3 times: bpr_epoch_any_kernel has 132 SMs x 8 CTAs x 128 = 135,168 threads
(450K steps = 3.3 passes); bpr_epoch_kernel has 67,584 quads at d <= 64 and 33,792 above.  For d >= 80, U, I and n are
halved, which keeps the isolated fraction, keeps each table at or under 1 GB (1M x 256 floats), and leaves 6.7 passes
of bpr_epoch_kernel at every d.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR, REG, STD = 0.05, 0.01, 0.1
FULL = (1_000_000, 2_000_000, 450_000)    # users with feedback, items, steps
HALF = (500_000, 1_000_000, 225_000)
N_EMPTY = 1000                            # users without feedback, appended after the others

QUAD_ROUND = [16, 32, 64, 128]    # the one-launch round kernel (ATOMIC), the pipelined kernel (STORE)
QUAD_DYN = [48, 80, 256]          # the two-pass quad path
SCALAR = [3, 8, 10, 24, 40]       # one thread per triple: tail only (3), the 8-wide block (8, 10, 24, 40)


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


_data = {}


def dataset(size):
    """(off, items, n_steps) with N_EMPTY users without feedback after the others; built once per size."""
    if size not in _data:
        from gorse_b200 import synth

        U, I, n = size
        off, items = synth.make_feedback(U, I, 2 * U, seed=31, zipf_s=0.0)
        off = np.concatenate([off, np.full(N_EMPTY, off[-1])]).astype(np.int64)
        _data[size] = (off, items, I, n)
    return _data[size]


def start(U, I, d, seed):
    rng = np.random.default_rng(seed)
    P = rng.standard_normal((U, d), dtype=np.float32) * np.float32(STD)
    Q = rng.standard_normal((I, d), dtype=np.float32) * np.float32(STD)
    return P, Q


def isolated(uij, U, I):
    """Mask of the live triples that share no user and no item with another live triple, and the masks of the user
    and item rows some live triple touches."""
    live = uij[:, 2] >= 0
    u, i, j = uij[live, 0], uij[live, 1], uij[live, 2]
    cu = np.bincount(u, minlength=U)
    ci = np.bincount(np.concatenate([i, j]), minlength=I)
    iso = np.zeros(len(uij), bool)
    iso[live] = (cu[u] == 1) & (ci[i] == 1) & (ci[j] == 1)
    return iso, cu > 0, ci > 0


def check_epoch(gb, orc, m, U, I, d, n, seed, scatter, P0, Q0):
    """Run one epoch of n steps and check it on the isolated triples; returns their number."""
    uij = m.bpr_sample_triples(seed=seed, first_step=0, n=n) if n else np.zeros((0, 3), np.int32)
    m.bpr_epoch(LR, REG, n, seed, scatter)
    Pg, Qg = m.get_factors()
    iso, touched_u, touched_i = isolated(uij, U, I)
    t = uij[iso]
    k = len(t)
    # the oracle on a compact sub-problem: row k of Pc is the user of isolated triple k, rows k and k + K of Qc its items
    Pc = np.ascontiguousarray(P0[t[:, 0]])
    Qc = np.ascontiguousarray(np.concatenate([Q0[t[:, 1]], Q0[t[:, 2]]]))
    if k:
        ids = np.arange(k, dtype=np.int32)
        orc.bpr_apply_triples(Pc, Qc, np.stack([ids, ids, ids + k], 1), LR, REG)
    got_p, got_q = Pg[t[:, 0]], np.concatenate([Qg[t[:, 1]], Qg[t[:, 2]]])
    before_p, before_q = P0[t[:, 0]], np.concatenate([Q0[t[:, 1]], Q0[t[:, 2]]])
    for got, want, before in ((got_p, Pc, before_p), (got_q, Qc, before_q)):
        if scatter == gb.SCATTER_STORE:
            assert got.tobytes() == want.tobytes()
        else:
            bound = 2 * np.spacing(np.abs(before) + np.abs(want)).astype(np.float64)
            err = np.abs(got.astype(np.float64) - want)
            assert (err <= bound).all(), (err.max(), np.unravel_index(np.argmax(err - bound), err.shape))
    for got, before, touched in ((Pg, P0, touched_u), (Qg, Q0, touched_i)):
        assert np.isfinite(got).all()
        moved = (got.view(np.uint32) != before.view(np.uint32)).any(1)
        assert not moved[~touched].any()
    if k:
        assert not np.array_equal(got_q, before_q)
    return k


@pytest.mark.parametrize("d", QUAD_ROUND + QUAD_DYN + SCALAR)
@pytest.mark.parametrize("scatter", ["store", "atomic"])
def test_isolated_triples_match_oracle(gb, orc, ctx, scatter, d):
    size = HALF if d >= 80 else FULL
    off, items, I, n = dataset(size)
    U = len(off) - 1
    P0, Q0 = start(U, I, d, seed=d)
    mode = gb.SCATTER_STORE if scatter == "store" else gb.SCATTER_ATOMIC
    with gb.CFModel(ctx, U, I, d, off, items) as m:
        m.set_factors(P0, Q0)
        k = check_epoch(gb, orc, m, U, I, d, n, 1000 + d, mode, P0, Q0)
    assert k >= 10_000


@pytest.mark.parametrize("n", [0, 1, 65, 8193])
@pytest.mark.parametrize("d", [16, 48, 10])
@pytest.mark.parametrize("scatter", ["store", "atomic"])
def test_short_epochs(gb, orc, ctx, scatter, d, n):
    """An empty epoch, one step, a partial CTA, and one round plus one step.  At 8193 steps over these U and I, ~93 % of
    the triples are isolated."""
    from gorse_b200 import synth

    U, I = 200_000, 1_000_000
    off, items = synth.make_feedback(U, I, 2 * U, seed=32, zipf_s=0.0)
    P0, Q0 = start(U, I, d, seed=5)
    mode = gb.SCATTER_STORE if scatter == "store" else gb.SCATTER_ATOMIC
    with gb.CFModel(ctx, U, I, d, off, items) as m:
        m.set_factors(P0, Q0)
        seed = 7
        while n and (m.bpr_sample_triples(seed=seed, first_step=0, n=1)[0, 2] < 0):
            seed += 1   # a first step with a valid negative, so that n = 1 updates something
        k = check_epoch(gb, orc, m, U, I, d, n, seed, mode, P0, Q0)
    assert k >= 0.8 * n


@pytest.mark.parametrize("d", [16, 48, 10])
@pytest.mark.parametrize("scatter", ["store", "atomic"])
def test_dead_stream_changes_nothing(gb, ctx, scatter, d):
    """Every user holds every item, so no triple has a valid negative (j = -1) and the epoch must leave the tables
    bit-identical: the only check of the live flag in the store pipeline and of the skipped entries of the rounds."""
    U, I = 3000, 24
    off = (np.arange(U + 1, dtype=np.int64) * I)
    items = np.tile(np.arange(I, dtype=np.int32), U)
    P0, Q0 = start(U, I, d, seed=9)
    mode = gb.SCATTER_STORE if scatter == "store" else gb.SCATTER_ATOMIC
    n = 3 * 8192 + 77
    with gb.CFModel(ctx, U, I, d, off, items) as m:
        assert (m.bpr_sample_triples(seed=3, first_step=0, n=1000)[:, 2] == -1).all()
        m.set_factors(P0, Q0)
        m.bpr_epoch(LR, REG, n, 3, mode)
        Pg, Qg = m.get_factors()
    assert Pg.tobytes() == P0.tobytes() and Qg.tobytes() == Q0.tobytes()
