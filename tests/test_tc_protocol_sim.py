"""Discrete-event model of the mbarrier protocols of the Hopper tensor-core kernels (csrc/conv1d_tc.cu, csrc/conv1d_gp.cu,
csrc/resblock_gp.cu).

Both deadlocks of round 1 were protocol bugs that a GPU can only show as a hang (producer groups running two ring phases
ahead of a parity wait; a consumer releasing a buffer it never waited for).  This model replays the kernels' role loops --
producers (in groups) or bulk-copy loader + transform warps, weight loader, the eight consumer warps -- as coroutines over
barriers with the hardware's semantics (arrival count, phase bit, `try_wait.parity(P)` passes iff the current phase parity
!= P; a wgmma reads its shared-memory operands until `wgmma.wait_group` has seen it complete, which the consumers do one
step after issuing it) under many random schedules, and checks: no deadlock, every slot holds the expected contents when it
is read, no slot is overwritten before its last reader is done.  The role loops are transcribed from the kernels (for the two
granule-planar kernels, from the roles they share in csrc/gp_pipeline.cuh: one model of the x loader and the transform warps,
and `mma_steps` for the consumers' tap chains with their one-behind release); the planner (ring depths, groups) is the real one.
"""
import ctypes
import random

import pytest

from emotivoice_b200 import _abi

NCONS_WARPS = 8
NPWARPS = 6


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0, "more arrivals than the barrier expects in one phase"
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def passes(self, parity):
        return (self.phase & 1) != parity


class Sim:
    """Cooperative scheduler.  Roles are generators yielding ('wait', bar, parity) | ('arrive', bar) | ('write', slot, tag)
    | ('read', slot, tag); a random runnable role advances each step."""

    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.slots = {}
        self.roles = []

    def add(self, name, gen):
        self.roles.append([name, gen, None])

    def run(self, max_steps=2_000_000):
        live = list(self.roles)
        for _ in range(max_steps):
            if not live:
                return
            runnable = [r for r in live if r[2] is None or r[2][0].passes(r[2][1])]
            if not runnable:
                raise AssertionError("deadlock: %r" % ([(r[0], r[2][1], r[2][0].phase) for r in live],))
            role = self.rng.choice(runnable)
            name, gen = role[0], role[1]
            role[2] = None
            try:
                ev = next(gen)
            except StopIteration:
                live.remove(role)
                continue
            kind = ev[0]
            if kind == "wait":
                role[2] = (ev[1], ev[2])
            elif kind == "arrive":
                ev[1].arrive()
            elif kind == "write":
                self.slots[ev[1]] = ev[2]
            elif kind == "read":
                assert self.slots.get(ev[1]) == ev[2], "%s read %s: holds %r, expected %r" % (name, ev[1], self.slots.get(ev[1]), ev[2])
        raise AssertionError("simulation did not finish")


def mma_steps(steps, b_empty, early_release=False):
    """A consumer warp's main loop over `steps` = [(wait_list, reads, releases)]: wait for the step's operands, issue its MMAs, then
    (wgmma.wait_group 1) the PREVIOUS step's MMAs have completed -- their operand reads happen up to here -- and its stages are handed
    back.  early_release: the bug the kernels must not have, releasing a step's stages at issue, before its MMAs have read them."""
    prev = None
    for waits, reads, releases in steps:
        for bar, parity in waits:
            yield ("wait", bar, parity)
        if early_release:
            for bar in releases:
                yield ("arrive", bar)
        if prev is not None:
            for slot, tag in prev[0]:
                yield ("read", slot, tag)
            if not early_release:
                for bar in prev[1]:
                    yield ("arrive", bar)
        prev = (reads, releases)
    if prev is not None:                                       # wgmma.wait_group 0
        for slot, tag in prev[0]:
            yield ("read", slot, tag)
        if not early_release:
            for bar in prev[1]:
                yield ("arrive", bar)


# ------------------------------------------------------------------------------------------------------------------
# conv1d_tc.cu
# ------------------------------------------------------------------------------------------------------------------
def sim_conv(seed, tiles, n_cb, K, a_stages, b_stages, ngroups, early_release=False):
    """tiles: list of booleans (True = active tile, False = padding tile that every role skips)."""
    sim = Sim(seed)
    wpg = NPWARPS // ngroups
    a_full = [Bar(wpg) for _ in range(a_stages)]            # one arrival per producer warp here (the kernel: per thread)
    a_empty = [Bar(NCONS_WARPS) for _ in range(a_stages)]
    b_full = [Bar(1) for _ in range(b_stages)]
    b_empty = [Bar(NCONS_WARPS) for _ in range(b_stages)]

    def producer(grp, w):
        a_cnt = 0
        for ti, active in enumerate(tiles):
            if not active:
                continue
            for cb in range(n_cb):
                if a_cnt % ngroups == grp:
                    s = a_cnt % a_stages
                    yield ("wait", a_empty[s], ((a_cnt // a_stages) & 1) ^ 1)
                    if w == 0:
                        yield ("write", ("A", s), (ti, cb))
                    yield ("arrive", a_full[s])
                a_cnt += 1

    def loader():
        b_cnt = 0
        for ti, active in enumerate(tiles):
            if not active:
                continue
            for cb in range(n_cb):
                for j in range(K):
                    sb = b_cnt % b_stages
                    yield ("wait", b_empty[sb], ((b_cnt // b_stages) & 1) ^ 1)
                    yield ("write", ("B", sb), (ti, cb, j))
                    yield ("arrive", b_full[sb])           # expect_tx + complete_tx of the bulk copy
                    b_cnt += 1

    def consumer():
        a_cnt = b_cnt = 0
        for ti, active in enumerate(tiles):
            if not active:
                continue
            steps = []
            for cb in range(n_cb):
                sa = a_cnt % a_stages
                for j in range(K):
                    sb = b_cnt % b_stages
                    waits = ([(a_full[sa], (a_cnt // a_stages) & 1)] if j == 0 else []) + [(b_full[sb], (b_cnt // b_stages) & 1)]
                    steps.append((waits, [(("A", sa), (ti, cb)), (("B", sb), (ti, cb, j))],
                                  [b_empty[sb]] + ([a_empty[sa]] if j == K - 1 else [])))
                    b_cnt += 1
                a_cnt += 1
            yield from mma_steps(steps, b_empty, early_release)

    for g in range(ngroups):
        for w in range(wpg):
            sim.add("producer%d.%d" % (g, w), producer(g, w))
    sim.add("loader", loader())
    for w in range(NCONS_WARPS):
        sim.add("consumer%d" % w, consumer())
    sim.run()


def _tc_plan(lib, B, L, Cin, Cout, K, dil, mode, ksplit=0):
    v = (ctypes.c_int * 11)()
    assert lib.ev_debug_tc_plan(B, L, Cin, Cout, K, dil, mode, ksplit, v) == 0
    return dict(zip("BN MT KBG a_stages b_stages groups ksplit acc smem tiles rows_pad".split(), list(v)))


@pytest.fixture(scope="module")
def lib():
    from emotivoice_b200 import build
    build.build(verbose=False)
    return _abi.load()


@pytest.mark.parametrize("shape", [(1, 537, 384, 1152, 1, 1), (1, 537, 1536, 384, 3, 1), (1, 34368, 128, 128, 11, 5),
                                   (1, 137472, 32, 32, 3, 1), (1, 4296, 256, 256, 7, 3), (1, 100, 384, 384, 3, 1)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_conv_protocol_with_the_real_plans(lib, shape, mode):
    B, L, Cin, Cout, K, dil = shape
    pl = _tc_plan(lib, B, L, Cin, Cout, K, dil, mode)
    cpg = 8 if mode == 2 else 4
    n_cb = -(-Cin // (cpg * pl["KBG"]))
    for seed in range(6):
        rng = random.Random(seed)
        tiles = [rng.random() > 0.2 for _ in range(rng.randint(1, 5))]       # tiles of ONE persistent CTA, some of them padding
        sim_conv(seed, tiles, n_cb, K, pl["a_stages"], pl["b_stages"], pl["groups"])


def test_conv_protocol_model_catches_the_round1_bugs():
    """The model is only worth something if it fails on the protocol that hung the GPU in round 1 and on a consumer that hands a
    stage back before its MMAs have read it."""
    with pytest.raises(AssertionError):                       # 6 producer groups on a 2-deep ring: parity cannot tell phases apart
        for seed in range(20):
            sim_conv(seed, [True, True, True], n_cb=12, K=3, a_stages=2, b_stages=4, ngroups=6)
    with pytest.raises(AssertionError):                       # stages released at issue, before wgmma.wait_group
        for seed in range(50):
            sim_conv(seed, [True] * 6, n_cb=2, K=3, a_stages=2, b_stages=2, ngroups=2, early_release=True)


# ------------------------------------------------------------------------------------------------------------------
# gp_pipeline.cuh (conv1d_gp.cu, resblock_gp.cu): x loader (bulk copies) -> a_full -> transform warps (in place) -> a_ready ->
# MMA -> a_empty -> x loader
# ------------------------------------------------------------------------------------------------------------------
NTW = 4


def add_x_roles(sim, tiles, n_cb, a_stages):
    """The x loader (load_x_tile) and the four transform warps (transform_tile) over `tiles` (booleans: False = a padding tile that
    every role skips); returns the barriers the consumers wait on and release, a_ready and a_empty.  Slot ("A", s) holds
    ("raw", tile, block) once the bulk copies land and ("op", tile, block) once transformed."""
    a_full = [Bar(1) for _ in range(a_stages)]
    a_ready = [Bar(NTW) for _ in range(a_stages)]           # one arrival per transform warp here (the kernel: per thread)
    a_empty = [Bar(NCONS_WARPS) for _ in range(a_stages)]

    def aloader():
        a_cnt = 0
        for ti, active in enumerate(tiles):
            if not active:
                continue
            for cb in range(n_cb):
                s = a_cnt % a_stages
                yield ("wait", a_empty[s], ((a_cnt // a_stages) & 1) ^ 1)
                yield ("write", ("A", s), ("raw", ti, cb))       # expect_tx + the bulk copies' complete_tx
                yield ("arrive", a_full[s])
                a_cnt += 1

    def xform(w):
        a_cnt = 0
        for ti, active in enumerate(tiles):
            if not active:
                continue
            for cb in range(n_cb):
                s = a_cnt % a_stages
                yield ("wait", a_full[s], (a_cnt // a_stages) & 1)
                if w == 0:
                    yield ("read", ("A", s), ("raw", ti, cb))
                    yield ("write", ("A", s), ("op", ti, cb))
                yield ("arrive", a_ready[s])
                a_cnt += 1

    sim.add("aloader", aloader())
    for w in range(NTW):
        sim.add("xform%d" % w, xform(w))
    return a_ready, a_empty


# ------------------------------------------------------------------------------------------------------------------
# conv1d_gp.cu: per tile, K taps per channel block
# ------------------------------------------------------------------------------------------------------------------
def sim_gp(seed, tiles, n_cb, K, a_stages, b_stages, early_release=False):
    """tiles: list of booleans (True = active tile, False = padding tile that every role skips); K: taps, or taps per tile (a
    grouped launch)."""
    sim = Sim(seed)
    taps = (lambda ti: K[ti]) if isinstance(K, (list, tuple)) else (lambda ti: K)     # grouped launch: the taps differ from tile to tile
    a_ready, a_empty = add_x_roles(sim, tiles, n_cb, a_stages)
    b_full = [Bar(1) for _ in range(b_stages)]
    b_empty = [Bar(NCONS_WARPS) for _ in range(b_stages)]

    def bloader():
        b_cnt = 0
        for ti, active in enumerate(tiles):
            if not active:
                continue
            for cb in range(n_cb):
                for j in range(taps(ti)):
                    sb = b_cnt % b_stages
                    yield ("wait", b_empty[sb], ((b_cnt // b_stages) & 1) ^ 1)
                    yield ("write", ("B", sb), (ti, cb, j))
                    yield ("arrive", b_full[sb])
                    b_cnt += 1

    def consumer():
        a_cnt = b_cnt = 0
        for ti, active in enumerate(tiles):
            if not active:
                continue
            steps = []
            for cb in range(n_cb):
                sa = a_cnt % a_stages
                for j in range(taps(ti)):
                    sb = b_cnt % b_stages
                    waits = ([(a_ready[sa], (a_cnt // a_stages) & 1)] if j == 0 else []) + [(b_full[sb], (b_cnt // b_stages) & 1)]
                    steps.append((waits, [(("A", sa), ("op", ti, cb)), (("B", sb), (ti, cb, j))],
                                  [b_empty[sb]] + ([a_empty[sa]] if j == taps(ti) - 1 else [])))
                    b_cnt += 1
                a_cnt += 1
            yield from mma_steps(steps, b_empty, early_release)

    sim.add("bloader", bloader())
    for w in range(NCONS_WARPS):
        sim.add("consumer%d" % w, consumer())
    sim.run()


def _gp_plan(lib, B, L, Cin, Cout, K, dil, rate, mode):
    v = (ctypes.c_int * 11)()
    assert lib.ev_debug_gp_plan(B, L, Cin, Cout, K, dil, rate, mode, v) == 0, lib.ev_last_error()
    return dict(zip("BN MT KBG a_stages b_stages ntw planes acc smem tiles rows_pad".split(), list(v)))


GP_SHAPES = [(1, 537, 80, 512, 7, 1, 1), (1, 537, 512, 2048, 3, 1, 8), (1, 4296, 256, 256, 11, 5, 1), (1, 34368, 128, 128, 11, 1, 1),
             (1, 34368, 128, 128, 3, 1, 2), (1, 68736, 64, 64, 7, 3, 1), (1, 137472, 32, 32, 3, 1, 1), (32, 262144, 32, 32, 11, 5, 1),
             (8, 65536, 128, 128, 11, 5, 1), (128, 32768, 256, 256, 7, 1, 1)]


@pytest.mark.parametrize("shape", GP_SHAPES)
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_gp_plans_respect_the_hardware_limits_and_the_protocol(lib, shape, mode):
    B, L, Cin, Cout, K, dil, rate = shape
    pl = _gp_plan(lib, B, L, Cin, Cout, K, dil, rate, mode)
    cpg = 8 if mode == 2 else 4
    assert pl["smem"] <= 227 * 1024 and 2 <= pl["a_stages"] <= 8 and 1 <= pl["b_stages"] <= 8
    assert pl["acc"] == pl["MT"] * pl["BN"] <= 128        # register accumulators: MT x BN columns x 64 rows per consumer warpgroup
    assert pl["BN"] % 32 == 0 and Cout % pl["BN"] == 0 and pl["planes"] == (2 if mode == 1 else 1)
    rows = 128 * pl["MT"] + (K - 1) * dil
    assert pl["rows_pad"] >= rows and pl["rows_pad"] % 8 == 0
    # one stage's transaction count must fit the mbarrier tx-count field (2^20 - 1 bytes)
    assert pl["KBG"] * pl["rows_pad"] * 16 < (1 << 20) and pl["planes"] * pl["KBG"] * pl["BN"] * 16 < (1 << 20)
    n_cb = -(-Cin // (cpg * pl["KBG"]))
    for seed in range(5):
        rng = random.Random(seed)
        tiles = [rng.random() > 0.2 for _ in range(rng.randint(1, 5))]
        sim_gp(seed, tiles, min(n_cb, 6), K, pl["a_stages"], pl["b_stages"])


def test_gp_summation_order_parameters_do_not_depend_on_batch_or_length(lib):
    """KBG (channels per pipeline stage) fixes the order of each output element's reduction: it must be a function of the
    layer shape only, or a batch would not be bitwise equal to its items' B=1 runs."""
    for (Cin, Cout, K, dil, rate) in [(80, 512, 7, 1, 1), (512, 2048, 3, 1, 8), (256, 256, 11, 5, 1), (128, 128, 7, 3, 1), (32, 32, 11, 5, 1)]:
        for mode in (0, 1, 2):
            kbgs = {_gp_plan(lib, B, L, Cin, Cout, K, dil, rate, mode)["KBG"] for (B, L) in [(1, 64), (1, 5000), (3, 70000), (32, 300000)]}
            assert len(kbgs) == 1, (Cin, Cout, K, dil, mode, kbgs)


def _gp_group_plan(lib, Ks, dils, B, L, Cin, Cout, mode):
    n = len(Ks)
    v = (ctypes.c_int * 11)()
    IA = ctypes.c_int * n
    assert lib.ev_debug_gp_group_plan(n, IA(*Ks), IA(*dils), B, L, Cin, Cout, mode, v) == 0, lib.ev_last_error()
    return dict(zip("BN MT KBG a_stages b_stages ntw planes acc smem tiles rows_pad".split(), list(v)))


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("shape", [(1, 4296, 256), (1, 34368, 128), (2, 3000, 128), (3, 900, 64)])
def test_gp_grouped_launch_plans(lib, shape, mode):
    """The grouped launch (three convolutions of one shape in a kernel) must use each member's own K granules per stage (the
    reduction order: bitwise equality with the members' own launches), size its stages for the widest halo, and carry every
    member's tiles; and it must fit the same hardware limits as a single launch."""
    B, L, C = shape
    Ks, dils = (3, 7, 11), (1, 3, 5)
    g = _gp_group_plan(lib, Ks, dils, B, L, C, C, mode)
    solo = [_gp_plan(lib, B, L, C, C, K, d, 1, mode) for K, d in zip(Ks, dils)]
    assert {p["KBG"] for p in solo} == {g["KBG"]}
    assert g["smem"] <= 227 * 1024 and g["acc"] == g["MT"] * g["BN"] <= 128
    assert g["rows_pad"] >= 128 * g["MT"] + (11 - 1) * 5 and g["rows_pad"] % 8 == 0
    tiles_one = B * -(-L // (128 * g["MT"])) * (C // g["BN"])
    assert g["tiles"] == 3 * tiles_one
    n_cb = -(-C // ((8 if mode == 2 else 4) * g["KBG"]))
    for seed in range(3):
        rng = random.Random(seed)
        n = rng.randint(2, 6)
        sim_gp(seed, [True] * n, min(n_cb, 4), [rng.choice(Ks) for _ in range(n)], g["a_stages"], g["b_stages"])


@pytest.mark.parametrize("mode", [0, 2, 3])
@pytest.mark.parametrize("C,mul", [(256, 8), (128, 64)])
def test_gp_grouped_launch_plans_over_utterance_lengths(lib, C, mul, mode):
    """The grouped convolution plan over every length a batch-1 step can have: members' own K granules, all tiles carried, limits kept."""
    for F in range(40, 2401, 17):
        L = F * mul
        g = _gp_group_plan(lib, (3, 7, 11), (1, 3, 5), 1, L, C, C, mode)
        assert g["KBG"] == _gp_plan(lib, 1, L, C, C, 11, 5, 1, mode)["KBG"] == _gp_plan(lib, 1, L, C, C, 3, 1, 1, mode)["KBG"]
        assert g["tiles"] == 3 * -(-L // (128 * g["MT"])) * (C // g["BN"]) and g["MT"] in (1, 2, 4)
        assert g["smem"] <= 227 * 1024 and g["acc"] == g["MT"] * g["BN"] <= 128 and g["rows_pad"] >= 128 * g["MT"] + 50


def test_gp_grouped_launch_plan_fills_the_machine_at_batch_1(lib):
    """HiFi-GAN stage 1 at batch 1 in the fp32 mode: 3 x 68 one-accumulator tiles (204 > 132 SMs) instead of 3 x 34 two-accumulator
    ones -- the plan is picked by simulating the round-robin deal, where the k = 11 member's double tile would be the critical path."""
    g = _gp_group_plan(lib, (3, 7, 11), (1, 3, 5), 1, 4296, 256, 256, 3)
    assert g["MT"] == 1 and g["tiles"] == 204


def test_gp_grouped_launch_protocol():
    """A grouped launch (conv1d_gp_group: the same-index convolutions of three parallel ResBlocks in one kernel) changes the number of
    taps -- weight stages per activation stage -- from tile to tile; the weight loader and the MMA issuer derive it from the same
    tile decode, so the rings stay in step for any mix and any ring depth."""
    for seed in range(30):
        rng = random.Random(seed)
        n = rng.randint(2, 7)
        tiles = [rng.random() > 0.15 for _ in range(n)]
        taps = [rng.choice((3, 7, 11)) for _ in range(n)]
        sim_gp(seed, tiles, rng.randint(1, 4), taps, rng.randint(2, 4), rng.randint(2, 8))


@pytest.mark.parametrize("mode", [0, 2, 3])
@pytest.mark.parametrize("C,mul", [(64, 128), (32, 256)])
def test_resblock_gp_grouped_launch_plans_over_utterance_lengths(lib, C, mul, mode):
    """Host logic of the grouped fused launch over the lengths a batch-1 step can have (every frame count from 40 to 2400 in steps of
    13): members in launch order heaviest first, each with ITS OWN rows per tile R = 128 MT - (K - 1) and row-tile count, tile
    ranges contiguous and complete, stage sizes for the widest halo, hardware limits respected.  A wrong first-tile index or tile
    count would make the roles of the kernel walk different tile sequences (a hang), so this is checked here, on the CPU."""
    Ks, dils = (3, 7, 11), (1, 3, 5)
    IA = ctypes.c_int * 3
    seen_mt = set()
    for F in range(40, 2401, 13):
        L = F * mul
        v = (ctypes.c_int * 16)()
        rc = lib.ev_debug_resblock_gp_group_plan(3, IA(*Ks), IA(*dils), 1, L, C, mode, v)
        solo = []
        for K, d in zip(Ks, dils):
            w = (ctypes.c_int * 11)()
            solo.append(list(w) if lib.ev_debug_resblock_gp_plan(1, L, C, K, d, mode, w) == 0 else None)
        if any(x is None or x[0] < 2 for x in solo):
            assert rc != 0          # a member that would not be fused on its own is never grouped
            continue
        assert rc == 0, lib.ev_last_error()
        mt, kbg, total, rows1_pad, rows2_pad, smem, acc = list(v)[:7]
        members = [tuple(v[7 + 3 * i: 10 + 3 * i]) for i in range(3)]
        seen_mt.add(mt)
        assert mt in (2, 4) and {x[1] for x in solo} == {kbg}
        assert [m[0] for m in members] == [11, 7, 3]                      # heaviest first
        t0 = 0
        for K, tiles_m, tile0 in members:
            R = 128 * mt - (K - 1)
            assert tiles_m == -(-L // R) and tile0 == t0
            t0 += tiles_m
        assert total == t0
        assert rows1_pad >= 128 * mt + 10 * 5 and rows2_pad >= 128 * mt + 10 and rows1_pad % 8 == 0 and rows2_pad % 8 == 0
        assert smem <= 227 * 1024 and acc == mt * C <= 128
    assert seen_mt


def test_resblock_gp_grouped_launch_protocol():
    """Grouped fused-ResBlock launch: consecutive tiles of a CTA may belong to layers with different taps; the weight loader streams
    w1 then w2 of each tile's own layer, exactly as the consumers read them."""
    for seed in range(30):
        rng = random.Random(seed)
        n = rng.randint(1, 6)
        sim_pair(seed, n, rng.randint(1, 3), [rng.choice((3, 7, 11)) for _ in range(n)], rng.randint(2, 4), rng.randint(2, 8))


def test_gp_protocol_model_is_sensitive():
    """The model must fail when the consumers hand a stage back before wgmma.wait_group has seen the MMAs that read it complete
    (the conv1d_gp and fused-ResBlock consumers release one step behind the issue for that reason)."""
    with pytest.raises(AssertionError):
        for seed in range(40):
            sim_gp(seed, [True] * 5, n_cb=2, K=3, a_stages=2, b_stages=2, early_release=True)
    with pytest.raises(AssertionError):
        for seed in range(40):
            sim_pair(seed, 3, 2, 3, 2, 2, early_release=True)


# ------------------------------------------------------------------------------------------------------------------
# resblock_gp.cu: per tile c1 -> epi1 (xt tile in shared memory) -> c2 -> epi2, all in the consumer warps
# ------------------------------------------------------------------------------------------------------------------
def sim_pair(seed, n_tiles, n_cb, K, a_stages, b_stages, early_release=False):
    """Per tile, every consumer warp runs c1 over the x ring, epi1 into the shared xt tile between two named barriers of the eight
    consumer warps (the first: both warpgroups' c2 of the previous tile have read the tile; the second: it is complete), then c2
    over the xt tile; the weight loader streams w1 then w2 of every tile."""
    sim = Sim(seed)
    taps = (lambda ti: K[ti]) if isinstance(K, (list, tuple)) else (lambda ti: K)     # grouped launch: the taps differ from tile to tile
    a_ready, a_empty = add_x_roles(sim, [True] * n_tiles, n_cb, a_stages)
    b_full = [Bar(1) for _ in range(b_stages)]
    b_empty = [Bar(NCONS_WARPS) for _ in range(b_stages)]
    named = Bar(NCONS_WARPS)                                # bar.sync 1, 256

    def bloader():
        b_cnt = 0
        for ti in range(n_tiles):
            for which in (1, 2):
                for cb in range(n_cb):
                    for j in range(taps(ti)):
                        sb = b_cnt % b_stages
                        yield ("wait", b_empty[sb], ((b_cnt // b_stages) & 1) ^ 1)
                        yield ("write", ("B", sb), (which, ti, cb, j))
                        yield ("arrive", b_full[sb])
                        b_cnt += 1

    def consumer(w):
        a_cnt = b_cnt = uses = 0

        def bar_sync():
            nonlocal uses
            yield ("arrive", named)
            yield ("wait", named, uses & 1)
            uses += 1

        for ti in range(n_tiles):
            steps = []
            for cb in range(n_cb):
                sa = a_cnt % a_stages
                for j in range(taps(ti)):
                    sb = b_cnt % b_stages
                    waits = ([(a_ready[sa], (a_cnt // a_stages) & 1)] if j == 0 else []) + [(b_full[sb], (b_cnt // b_stages) & 1)]
                    steps.append((waits, [(("A", sa), ("op", ti, cb)), (("B", sb), (1, ti, cb, j))],
                                  [b_empty[sb]] + ([a_empty[sa]] if j == taps(ti) - 1 else [])))
                    b_cnt += 1
                a_cnt += 1
            yield from mma_steps(steps, b_empty, early_release)
            yield from bar_sync()
            yield ("write", ("A2", w), ti)                   # this warp's rows of the xt tile
            yield from bar_sync()
            steps = []
            for cb in range(n_cb):
                for j in range(taps(ti)):
                    sb = b_cnt % b_stages
                    reads = [(("A2", v), ti) for v in range(NCONS_WARPS)] + [(("B", sb), (2, ti, cb, j))]
                    steps.append(([(b_full[sb], (b_cnt // b_stages) & 1)], reads, [b_empty[sb]]))
                    b_cnt += 1
            yield from mma_steps(steps, b_empty, early_release)

    sim.add("bloader", bloader())
    for w in range(NCONS_WARPS):
        sim.add("consumer%d" % w, consumer(w))
    sim.run()


@pytest.mark.parametrize("C,K,dil", [(32, 3, 1), (32, 11, 5), (64, 7, 3), (64, 11, 5), (128, 11, 1)])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_resblock_gp_protocol_with_the_real_plans(lib, C, K, dil, mode):
    v = (ctypes.c_int * 11)()
    assert lib.ev_debug_resblock_gp_plan(1, 137472, C, K, dil, mode, v) == 0, lib.ev_last_error()
    pl = dict(zip("MT KBG a_stages b_stages ntw acc smem tiles R rows1_pad rows2_pad".split(), list(v)))
    assert pl["smem"] <= 227 * 1024 and pl["acc"] == pl["MT"] * C <= 128 and pl["a_stages"] >= 2 and pl["b_stages"] >= 2
    assert pl["R"] == 128 * pl["MT"] - (K - 1) and pl["rows1_pad"] >= 128 * pl["MT"] + (K - 1) * dil and pl["rows2_pad"] >= 128 * pl["MT"] + K - 1
    cpg = 8 if mode == 2 else 4
    n_cb = -(-C // (cpg * pl["KBG"]))
    for seed in range(5):
        sim_pair(seed, random.Random(seed).randint(1, 5), n_cb, K, pl["a_stages"], pl["b_stages"])


def test_resblock_gp_kbg_matches_the_unfused_kernel(lib):
    """The fused layer must reduce in the same order as the two launches it replaces: same channels per pipeline stage."""
    for C, K, dil in [(32, 3, 1), (32, 11, 5), (64, 7, 3), (64, 11, 5), (128, 11, 5)]:
        for mode in (0, 1, 2, 3):
            v, u = (ctypes.c_int * 11)(), (ctypes.c_int * 11)()
            assert lib.ev_debug_resblock_gp_plan(4, 50000, C, K, dil, mode, v) == 0
            assert lib.ev_debug_gp_plan(4, 50000, C, C, K, dil, 1, mode, u) == 0
            assert v[1] == u[2], (C, K, dil, mode)
