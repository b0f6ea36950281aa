"""CPU: discrete-event simulation of the mbarrier protocol of the fused renderer (csrc/render_fused_ws3.cu): its pass
schedule and the hand-off between its 24 warps - 12 gather, 8 decoder (two wgmma warpgroups), 4 ray.  Every role's control
flow is transcribed from the CUDA source (same loops, same barriers, parities and arrival counts, the same placement of
colours(n) and its two named barriers); work items get random durations and the runnable warps are stepped in random
order, over many seeds and group counts.  Asserted:
  * no deadlock and no lost mbarrier phase (a waiter that a barrier overtakes by two phases blocks forever);
  * A1 ring: the gather rewrites a stage only after all eight decoder warps have read its previous tile, and a decoder warp
    reads a stage only once all four warps of the team have written it;
  * colour areas (global workspace slices): CA[n % 3] is rewritten only after every decoder warp has read it in colours(n),
    FA only after colours(n - 1); colours(n) starts only after all eight decoder warps wrote all six of its tiles;
  * shared-memory hazards: the ray warps read a pass's sigma only after every decoder warp wrote its rows, a per-group state
    slot is not rewritten by the gather before its previous group is finished, the omega slot not before its previous
    group's colours are done, fine depths are read only after importance.
It mirrors the protocol, not the arithmetic; parity on hardware is what tests/test_render_gpu.py is for."""
import heapq
import random

import pytest

K_NA, K_EW, K_RW, K_TEAMS = 4, 8, 4, 3


def pass_at(j, N):                                   # render_fused_ws3.cu: pass_at
    if j == 0:
        return (0, 0)
    if N == 1:
        return (0, 1)
    if j == 1:
        return (1, 0)
    k, body = j - 2, 2 * (N - 2)
    if k < body:
        return ((k >> 1) + 2, 0) if (k & 1) else (k >> 1, 1)
    return (N - 2 + (k - body), 1)


def tile_at(q, N):
    j = q // 3
    n, p = pass_at(j, N)
    return (n, p, q - 3 * j)


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def passed(self, parity):                        # mbarrier.try_wait.parity
        return (self.phase & 1) != parity


class Sim:
    def __init__(self, N, seed, sig_count=K_EW):
        # sig_count: arrivals of sigc_ready / sigf_ready (the kernel: every decoder warp, K_EW); other values model a bug
        self.N, self.T, self.rng = N, 6 * N, random.Random(seed)
        B = Bar
        self.a1_full = [B(4) for _ in range(K_NA)]; self.a1_empty = [B(K_EW) for _ in range(K_NA)]
        self.fine_ready = [B(K_RW) for _ in range(4)]; self.state_free = [B(1) for _ in range(4)]
        self.sigc_ready = [B(sig_count) for _ in range(4)]; self.sigf_ready = [B(sig_count) for _ in range(4)]
        self.omega_ready = [B(K_RW) for _ in range(2)]
        self.now, self.events, self.seq = 0.0, [], 0
        # hazard bookkeeping
        self.a1_tile, self.a1_written, self.a1_read = [None] * K_NA, [0] * K_NA, [0] * K_NA
        self.area_owner = {}                          # colour area (CA, n % 3, k) | (FA, k) -> group
        self.area_writes = {}                         # (group, pass, k) -> decoder warps that stored their rows
        self.area_reads = {}                          # group -> decoder warps that finished reading it in colours()
        self.sigma_writes = {}                        # (group, pass) -> decoder warp-tiles that stored their sigma rows
        self.colours_done, self.importance_done, self.composite_done = set(), set(), set()
        self.state_owner = [None] * 4
        self.slot_owner = [None] * 2
        self.ebar_count, self.ebar_gen = 0, 0

    def dur(self, lo, hi):
        return self.rng.uniform(lo, hi)

    def later(self, dt, fn):
        self.seq += 1
        heapq.heappush(self.events, (self.now + dt, self.seq, fn))

    # ---------------------------------------------------------------- roles (generators yield ('wait', bar, parity) | ('work', dt) | ('ebar',))
    def gather_warp(self, gw):
        team, it = gw >> 2, 0
        for q in range(self.T):
            n, p, k = tile_at(q, self.N)
            my_it = it; it += 1
            if my_it % K_TEAMS != team:
                continue
            if p == 0:
                yield ('wait', self.state_free[n & 3], ((n >> 2) & 1) ^ 1)
                prev = self.state_owner[n & 3]
                assert prev is None or prev == n or prev in self.colours_done, f'state slot of group {prev} rewritten for {n}'
                self.state_owner[n & 3] = n
            else:
                yield ('wait', self.fine_ready[n & 3], (n >> 2) & 1)
                assert n in self.importance_done, f'fine gather of {n} before its importance sampling'
            stage = my_it % K_NA
            yield ('wait', self.a1_empty[stage], ((my_it // K_NA) & 1) ^ 1)
            if self.a1_tile[stage] != q:
                assert self.a1_tile[stage] is None or self.a1_read[stage] == K_EW, f'A1 stage {stage} rewritten before it was read'
                self.a1_tile[stage], self.a1_written[stage], self.a1_read[stage] = q, 0, 0
            yield ('work', self.dur(5, 20))
            self.a1_written[stage] += 1
            self.a1_full[stage].arrive()

    def decoder_warp(self, e):
        def colours(n):
            yield ('wait', self.omega_ready[n & 1], (n >> 1) & 1)
            assert n in self.composite_done and self.slot_owner[n & 1] == n
            assert all(self.area_writes.get((n, p, k), 0) == K_EW for p in (0, 1) for k in range(3)), f'colours({n}) before all six tiles'
            yield ('work', self.dur(1, 6))            # colour-area loads, shuffle reduction, shared-memory atomics
            self.area_reads[n] = self.area_reads.get(n, 0) + 1
            yield ('ebar',)
            yield ('work', self.dur(0.1, 0.5))
            yield ('ebar',)
            if e == 0:
                self.colours_done.add(n)
                self.state_free[n & 3].arrive()
        for it in range(self.T):
            n, p, k = tile_at(it, self.N)
            if p == 1 and k == 0 and n >= 1:
                yield from colours(n - 1)
            stage = it % K_NA
            yield ('wait', self.a1_full[stage], (it // K_NA) & 1)
            assert self.a1_tile[stage] == it and self.a1_written[stage] == 4, f'decoder reads A1 stage {stage} before tile {it} is complete'
            yield ('work', self.dur(0.5, 2))          # layer 1 (wgmma from shared memory)
            self.a1_read[stage] += 1
            self.a1_empty[stage].arrive()
            yield ('work', self.dur(1, 4))            # softplus, layer 2 from registers
            area = ('CA', n % 3, k) if p == 0 else ('FA', k)
            owner = self.area_owner.get(area)
            assert owner is None or owner == n or self.area_reads.get(owner, 0) == K_EW, \
                f'tile {(n, p, k)} overwrites {area} of group {owner} before colours({owner}) read it'
            self.area_owner[area] = n
            yield ('work', self.dur(0.2, 1))          # colour-area and sigma stores
            self.area_writes[(n, p, k)] = self.area_writes.get((n, p, k), 0) + 1
            self.sigma_writes[(n, p)] = self.sigma_writes.get((n, p), 0) + 1
            if k == 2:
                (self.sigc_ready if p == 0 else self.sigf_ready)[n & 3].arrive()
        yield from colours(self.N - 1)

    def ray_warp(self, rw):
        for j in range(2 * self.N):
            n, p = pass_at(j, self.N)
            si, par = n & 3, (n >> 2) & 1
            if p == 0:
                yield ('wait', self.sigc_ready[si], par)
                assert self.sigma_writes.get((n, 0), 0) == 3 * K_EW, f'importance({n}) before every coarse sigma was stored'
                yield ('work', self.dur(2, 12))
                if rw == 0:
                    self.importance_done.add(n)
                self.fine_ready[si].arrive()
            else:
                yield ('wait', self.sigf_ready[si], par)
                assert self.sigma_writes.get((n, 1), 0) == 3 * K_EW, f'composite({n}) before every fine sigma was stored'
                if n >= 2:
                    yield ('wait', self.state_free[(n - 2) & 3], ((n - 2) >> 2) & 1)
                    assert (n - 2) in self.colours_done
                prev = self.slot_owner[n & 1]
                assert prev is None or prev == n or prev in self.colours_done, f'omega slot of group {prev} rewritten for {n}'
                self.slot_owner[n & 1] = n
                yield ('work', self.dur(2, 12))
                if rw == 0:
                    self.composite_done.add(n)
                self.omega_ready[n & 1].arrive()

    def procs(self):
        return ([('G%d' % g, self.gather_warp(g)) for g in range(12)] + [('E%d' % e, self.decoder_warp(e)) for e in range(K_EW)] +
                [('R%d' % r, self.ray_warp(r)) for r in range(K_RW)])

    # ---------------------------------------------------------------- scheduler
    def run(self):
        procs = self.procs()
        state = {name: ('ready', None) for name, _ in procs}          # ready | wait(bar, parity) | sleep | ebar(gen) | done
        gens = dict(procs)

        def step(name):
            try:
                op = next(gens[name])
            except StopIteration:
                state[name] = ('done', None)
                return
            if op[0] == 'wait':
                state[name] = ('wait', (op[1], op[2]))
            elif op[0] == 'work':
                state[name] = ('sleep', None)
                self.later(op[1], lambda name=name: state.__setitem__(name, ('ready', None)))
            else:
                self.ebar_count += 1
                state[name] = ('ebar', self.ebar_gen)
                if self.ebar_count == K_EW:
                    self.ebar_count = 0
                    self.ebar_gen += 1
        guard = 0
        while True:
            guard += 1
            assert guard < 5_000_000
            runnable = []
            for name, (st, arg) in state.items():
                if st == 'ready' or (st == 'wait' and arg[0].passed(arg[1])) or (st == 'ebar' and arg != self.ebar_gen):
                    runnable.append(name)
            if runnable:
                step(self.rng.choice(runnable))
                continue
            if self.events:
                t, _, fn = heapq.heappop(self.events)
                self.now = t
                fn()
                continue
            break
        stuck = {n: s for n, s in state.items() if s[0] != 'done'}
        assert not stuck, f'deadlock with N={self.N}: {sorted(stuck)[:6]}'
        assert self.colours_done == set(range(self.N))


def test_pass_schedule_visits_every_group_once_in_a_valid_order():
    for N in range(1, 12):
        seq = [pass_at(j, N) for j in range(2 * N)]
        assert sorted(seq) == sorted([(n, p) for n in range(N) for p in (0, 1)])
        pos = {np_: i for i, np_ in enumerate(seq)}
        for n in range(N):
            assert pos[(n, 0)] < pos[(n, 1)]                                       # F(n) after C(n)
            if n + 1 < N:
                assert pos[(n, 1)] < pos[(n + 1, 1)] and pos[(n, 0)] < pos[(n + 1, 0)]
            if n + 3 < N:
                assert pos[(n + 1, 1)] < pos[(n + 3, 0)]                           # CA[n % 3] is free again before C(n+3)
            if N > 2 and 1 <= n and n + 1 < N:
                assert pos[(n + 1, 0)] < pos[(n, 1)]                               # >= one pass of slack for importance(n)


@pytest.mark.parametrize('N', [1, 2, 3, 4, 5, 7, 8, 13])
def test_protocol_has_no_deadlock_or_hazard(N):
    for seed in range(12):
        Sim(N, seed * 101 + N).run()


def test_simulation_catches_a_short_sigma_hand_off():
    """The model is not vacuous: with half the decoder warps counted on sigc_ready / sigf_ready (the arrival count of the
    earlier design, where four warps read sigma back) the ray warps start on sigma that is not all stored yet."""
    with pytest.raises(AssertionError, match='sigma was stored'):
        for seed in range(40):
            Sim(4, seed, sig_count=4).run()
