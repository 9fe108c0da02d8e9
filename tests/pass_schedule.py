"""TEST INFRASTRUCTURE ONLY -- a model of the CTA-pair exchange of `pointnet_pass_kernel<false>`
(points2surf_b200/csrc/net_tc.cu) and of the host code that launches it (`launch_pass`, `make_seg`).

This module mirrors the kernel and has to change with it: every function below restates one expression of net_tc.cu,
and `warpgroup` restates the per-query tile loop of one warpgroup (its `for (int qi = wg; ...)` loop) statement by
statement, as far as the schedule goes: which tile a step works on, whether it produces or receives it, the mbarrier
waits with the parities the kernel computes, the asynchronous stores into the peer's slot, the reads of its own slot,
the arrivals on the peer's `empty` barrier and the re-arm of its own `full` barrier.  The arithmetic is not modelled.

What the kernel does, in short.  CTA 2j and 2j + 1 of the grid form a cluster of two (`part` = the cluster rank) that
streams the queries q = stream + qi * nstreams; warpgroup wg of each CTA takes qi = wg, wg + 2, ...  A query has
tpq = s0.tiles + s1.tiles tiles of 64 points (segment 0 first).  Of each pair of tiles (2k, 2k + 1), the CTA whose `own`
bit selects it produces the tile (first and mid layers), stores its big-layer A fragments into the peer's receive slot
of the same warpgroup and runs its own big layer on them; at the odd step it receives the peer's tile of the pair.
For an odd tpq the last pair has one tile: the CTA that owns it produces it, the other only receives.  Running counts
of the tiles sent and received give the parities of the `empty` and `full` barriers.

`run_pair` executes the two warpgroups of one index (part 0 and part 1 of a cluster; the warpgroups of different
indices use separate slots and barriers and never interact) under a chosen interleaving, with mbarriers that follow
PTX's rules: an arrival or a complete_tx lands in the barrier's current phase, the phase completes when its pending
arrival count and its transaction count both reach zero, and a wait on parity p passes while the current phase's
parity differs from p.  A warpgroup is one agent: its 128 threads pass the exchange together (each tile's MMAs are
warpgroup-collective), so its 128 arrivals on `empty` are one arrival of 128.  `run_pair` raises ScheduleError when a
store lands in a slot whose previous tile has not been read, a read finds no tile or not the k-th one, a wait passes
before the arrival or store it waits for has landed or on a phase other than that one, or no agent can move before
both are done.
"""
import random

KTILE = 64                         # points per tile
KWG = 2                            # warpgroups per CTA
KSPLIT = 2                         # CTAs per query stream (Cfg<false>::kSplit): the cluster of two
SLOT_BYTES = 8 * 128 * 16          # Cfg<false>::kSlotBytes: 8 k-steps x 128 threads x 16 B of A fragments
EMPTY_COUNT = 128                  # the peer warpgroup's threads arrive on `empty` once they have read the slot


class ScheduleError(AssertionError):
    pass


# ---------------------------------------------------------------- host side (launch_pass, make_seg)
def seg_tiles(n):
    """make_seg: tiles of a segment of n points."""
    return (n + KTILE - 1) // KTILE if n > 0 else 0


def tiles_per_query(s0_tiles, s1_tiles):
    """launch_pass: p.tiles_per_query = s0.tiles + s1.tiles."""
    return s0_tiles + s1_tiles


def stream_count(B, pass_clusters):
    """launch_pass: streams = pass_clusters, at most B (grid = streams * kSplit)."""
    return min(pass_clusters, B)


def queries_of_stream(B, stream, nstreams):
    """Kernel: nq, the number of queries of a stream."""
    return (B - stream + nstreams - 1) // nstreams if B > stream else 0


def query_index(stream, qi, nstreams):
    """Kernel: q = stream + qi * nstreams."""
    return stream + qi * nstreams


# ---------------------------------------------------------------- kernel expressions
def own_tile(part, wg, qi):
    """Which tile of each pair this CTA's warpgroup produces for query qi: own = (part ^ wg ^ (qi >> 1)) & 1."""
    return (part ^ wg ^ (qi >> 1)) & 1


def step_tile(i, own):
    """The tile step i produces if it is this CTA's: tq = (i & ~1) + own."""
    return (i & ~1) + own


def is_mine(i, tq, tpq):
    """Step i produces (and sends) tile tq: mine = !(i & 1) && tq < tpq; otherwise it receives the peer's tile."""
    return (i & 1) == 0 and tq < tpq


def segment(i, tq, s0_tiles):
    """The segment a produced tile reads, and the tile's index inside it: sgi = tq < seg[0].tiles ? 0 : 1, local tile
    tq - (sgi ? seg[0].tiles : 0)."""
    sgi = 0 if tq < s0_tiles else 1
    return sgi, tq - (s0_tiles if sgi else 0)


# ---------------------------------------------------------------- one warpgroup's loop
def warpgroup(part, wg, nq, tpq):
    """The tile loop of warpgroup `wg` of CTA `part`, as a generator of the operations it performs in program order:
      ('produce', qi, i, tq)                  first and mid layers of tile tq at step i
      ('wait', bar, parity, tag)              mbar_wait_cluster_bounded on this CTA's `full` / `empty`; `tag` names the
                                              event the wait is for: ('send', k) = the peer's k-th store,
                                              ('recv', k) = the peer's arrival after its k-th read
      ('send', qi, tq, k)                     st_async of the tile into the peer's slot, complete_tx on the peer's full
      ('read', k)                             read of this CTA's slot, expected to hold the peer's k-th tile; the
                                              simulator sends back the tile as (qi, tq, k)
      ('arrive_empty', k)                     mbar_arrive_cluster on the peer's empty (128 threads)
      ('arm_full',)                           thread 0: arrive_expect_tx(full, kSlotBytes) for the next phase
      ('big', qi, i, tile)                    the big layer on `tile` = (query, tile index), into query qi's maxima
    Returns (nsend, nrecv)."""
    nsend = nrecv = 0
    for qi in range(wg, nq, KWG):
        own = own_tile(part, wg, qi)
        for i in range(tpq):
            tq = step_tile(i, own)
            if is_mine(i, tq, tpq):
                yield ('produce', qi, i, tq)
                if nsend > 0:
                    yield ('wait', 'empty', (nsend - 1) & 1, ('recv', nsend - 1))
                yield ('send', qi, tq, nsend)
                nsend += 1
                tile = (qi, tq)
            else:
                yield ('wait', 'full', nrecv & 1, ('send', nrecv))
                got = yield ('read', nrecv)
                yield ('arrive_empty', nrecv)
                yield ('arm_full',)
                nrecv += 1
                tile = got[:2]
            yield ('big', qi, i, tile)
    return nsend, nrecv


# ---------------------------------------------------------------- mbarrier and simulator
class MBarrier:
    """mbarrier.init count; arrive(.expect_tx); complete_tx; try_wait.parity.  `landed[tag]` = the phase in which the
    tagged arrival or complete_tx landed."""

    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0
        self.landed = {}

    def _land(self, tag):
        if tag is not None:
            self.landed[tag] = self.phase
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending, self.tx = self.count, 0

    def arrive(self, n=1, tx=0, tag=None):
        self.pending -= n
        self.tx += tx
        if self.pending < 0:
            raise ScheduleError('more arrivals than the barrier counts in one phase')
        self._land(tag)

    def complete_tx(self, nbytes, tag=None):
        self.tx -= nbytes
        if abs(self.tx) >= 1 << 20:
            raise ScheduleError('transaction count out of range')
        self._land(tag)

    def passes(self, parity):
        return (self.phase & 1) != parity


SCHEDULES = ('stores_land_at_once', 'stores_land_late', 'random')


def run_pair(wg, nq, tpq, schedule='random', seed=0):
    """Run part 0 and part 1 of warpgroup `wg` over nq queries of tpq tiles under one interleaving.
    schedule: 'stores_land_at_once' (a store lands before anything else moves, then part 0 before part 1),
    'stores_land_late' (part 1 before part 0, a store lands only when neither can move), 'random' (seeded).
    -> dict: 'produce' {part: [(qi, i, tq)]}, 'big' {part: [(qi, i, tile)]}, 'recv' {part: [(k, tile)]},
       'waits' [(part, bar, parity, phase)], 'counts' {part: (nsend, nrecv)}."""
    rng = random.Random(seed)
    full = [MBarrier(1), MBarrier(1)]
    empty = [MBarrier(EMPTY_COUNT), MBarrier(EMPTY_COUNT)]
    for p in (0, 1):                                   # kernel prologue, before the cluster barrier
        full[p].arrive(1, SLOT_BYTES)
    slot = [None, None]                                # the tile in each part's receive slot, or None once read
    flight = []                                        # stores issued and not landed: (destination part, tile)
    gens = [warpgroup(p, wg, nq, tpq) for p in (0, 1)]
    op, done = [None, None], [None, None]
    out = {'produce': {0: [], 1: []}, 'big': {0: [], 1: []}, 'recv': {0: [], 1: []}, 'waits': [], 'counts': {}}

    def advance(p, value=None):
        try:
            op[p] = gens[p].send(value) if op[p] is not None else next(gens[p])
        except StopIteration as e:
            op[p], done[p] = None, e.value

    def enabled(p):
        o = op[p]
        if o is None:
            return False
        if o[0] == 'wait':
            return (full if o[1] == 'full' else empty)[p].passes(o[2])
        return True

    def step(p):
        o, peer = op[p], p ^ 1
        kind = o[0]
        value = None
        if kind == 'produce':
            out['produce'][p].append(o[1:])
        elif kind == 'wait':
            bar = (full if o[1] == 'full' else empty)[p]
            ph = bar.landed.get(o[3])
            if ph is None:
                raise ScheduleError('part %d: wait on %s parity %d passed before %s landed' % (p, o[1], o[2], o[3]))
            if ph & 1 != o[2] or bar.phase != ph + 1:
                raise ScheduleError('part %d: wait on %s parity %d for %s, which landed in phase %d (barrier at phase %d)'
                                    % (p, o[1], o[2], o[3], ph, bar.phase))
            out['waits'].append((p, o[1], o[2], ph))
        elif kind == 'send':
            if slot[peer] is not None or any(d == peer for d, _ in flight):
                raise ScheduleError('part %d: store of tile %s into a slot that still holds an unread tile' % (p, o[1:]))
            flight.append((peer, o[1:]))
        elif kind == 'read':
            if slot[p] is None or slot[p][2] != o[1]:
                raise ScheduleError('part %d: read %d found %s in the slot' % (p, o[1], slot[p]))
            value, slot[p] = slot[p], None
            out['recv'][p].append((o[1], value))
        elif kind == 'arrive_empty':
            empty[peer].arrive(EMPTY_COUNT, tag=('recv', o[1]))
        elif kind == 'arm_full':
            full[p].arrive(1, SLOT_BYTES)
        elif kind == 'big':
            out['big'][p].append(o[1:])
        advance(p, value)

    def land(j):
        d, tile = flight.pop(j)
        if slot[d] is not None:
            raise ScheduleError('store of tile %s overwrote the unread tile %s' % (tile, slot[d]))
        slot[d] = tile
        full[d].complete_tx(SLOT_BYTES, tag=('send', tile[2]))

    advance(0)
    advance(1)
    while op[0] is not None or op[1] is not None or flight:
        agents = [p for p in ((1, 0) if schedule == 'stores_land_late' else (0, 1)) if enabled(p)]
        if schedule == 'stores_land_at_once':
            choice = ('land', 0) if flight else ('agent', agents[0]) if agents else None
        elif schedule == 'stores_land_late':
            choice = ('agent', agents[0]) if agents else ('land', 0) if flight else None
        else:
            choices = [('agent', p) for p in agents] + [('land', j) for j in range(len(flight))]
            choice = rng.choice(choices) if choices else None
        if choice is None:
            raise ScheduleError('deadlock: part 0 at %s, part 1 at %s' % (op[0], op[1]))
        if choice[0] == 'agent':
            step(choice[1])
        else:
            land(choice[1])
    if slot != [None, None]:
        raise ScheduleError('tiles left unread in the slots: %s' % slot)
    for p in (0, 1):
        if done[p][0] != done[p ^ 1][1]:
            raise ScheduleError('part %d sent %d tiles, part %d received %d' % (p, done[p][0], p ^ 1, done[p ^ 1][1]))
    out['counts'] = {0: done[0], 1: done[1]}
    return out
