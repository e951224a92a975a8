"""Protocol model of the fused ResBlock kernel's cross-tile consumer order (csrc/resblock_gp.cu), on the model of
tests/test_tc_protocol_sim.py.

The consumers run c2 of tile i into a second accumulator set, then c1 of tile i + 1 with the chunks of epi2(i) between its taps,
then epi1(i + 1) into the shared xt tile.  epi2 writes only global memory, so what the shared-memory protocol must still guarantee is
that epi1(i + 1) rewrites the xt tile only after BOTH warpgroups' c2(i) has read all of it (their taps read each other's rows):
the named barrier ahead of epi1.  The model replays the new order -- c2(i), wgmma.wait_group 0, then c1(i + 1) step by step with
an epi2(i) chunk after each tap -- against the real plans, and one adversarial variant without that barrier must fail.
"""
import ctypes
import random

import pytest

from test_tc_protocol_sim import NCONS_WARPS, Bar, Sim, add_x_roles, lib, mma_steps  # noqa: F401  (lib: the fixture)


def sim_pair_overlap(seed, n_tiles, n_cb, K, a_stages, b_stages, n_chunks=4, xt_barrier=True):
    sim = Sim(seed)
    taps = (lambda ti: K[ti]) if isinstance(K, (list, tuple)) else (lambda ti: K)
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

        def c1_under_epi2(ti):
            """c1(ti) in the kernel's order: issue a tap, wgmma.wait_group 1 (the previous tap's reads are done), hand its stages
            back, then one chunk of epi2(ti - 1) (global memory only: the model checks that it reads no shared slot)"""
            nonlocal a_cnt, b_cnt
            prev, q = None, 0
            for cb in range(n_cb):
                sa = a_cnt % a_stages
                for j in range(taps(ti)):
                    sb = b_cnt % b_stages
                    if j == 0:
                        yield ("wait", a_ready[sa], (a_cnt // a_stages) & 1)
                    yield ("wait", b_full[sb], (b_cnt // b_stages) & 1)
                    reads = [(("A", sa), ("op", ti, cb)), (("B", sb), (1, ti, cb, j))]
                    rel = [b_empty[sb]] + ([a_empty[sa]] if j == taps(ti) - 1 else [])
                    if prev is not None:
                        for slot, tag in prev[0]:
                            yield ("read", slot, tag)
                        for bar in prev[1]:
                            yield ("arrive", bar)
                    prev = (reads, rel)
                    if ti > 0 and q < n_chunks:
                        yield ("write", ("OUT", w, ti - 1, q), True)
                        q += 1
                    b_cnt += 1
                a_cnt += 1
            while ti > 0 and q < n_chunks:
                yield ("write", ("OUT", w, ti - 1, q), True)
                q += 1
            for slot, tag in prev[0]:                          # wgmma.wait_group 0
                yield ("read", slot, tag)
            for bar in prev[1]:
                yield ("arrive", bar)

        for ti in range(n_tiles):
            yield from c1_under_epi2(ti)
            if xt_barrier:
                yield from bar_sync()                          # both warpgroups' c2(ti - 1) have read the xt tile
            yield ("write", ("A2", w), ti)                     # epi1: this warp's rows of the xt tile
            yield from bar_sync()                              # the whole xt tile is written
            steps = []
            for cb in range(n_cb):
                for j in range(taps(ti)):
                    sb = b_cnt % b_stages
                    reads = [(("A2", v), ti) for v in range(NCONS_WARPS)] + [(("B", sb), (2, ti, cb, j))]
                    steps.append(([(b_full[sb], (b_cnt // b_stages) & 1)], reads, [b_empty[sb]]))
                    b_cnt += 1
            yield from mma_steps(steps, b_empty)               # c2(ti), ending in wgmma.wait_group 0
        for q in range(n_chunks):                              # the last tile's epi2, nothing in flight
            yield ("write", ("OUT", w, n_tiles - 1, q), True)

    sim.add("bloader", bloader())
    for w in range(NCONS_WARPS):
        sim.add("consumer%d" % w, consumer(w))
    sim.run()
    for w in range(NCONS_WARPS):
        for ti in range(n_tiles):
            for q in range(n_chunks):
                assert sim.slots.get(("OUT", w, ti, q)), "epi2 chunk %d of tile %d never stored by warp %d" % (q, ti, w)


@pytest.mark.parametrize("C,K,dil", [(32, 3, 1), (32, 11, 5), (64, 7, 3), (64, 11, 5), (128, 11, 1)])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_cross_tile_order_with_the_real_plans(lib, C, K, dil, mode):
    v = (ctypes.c_int * 11)()
    assert lib.ev_debug_resblock_gp_plan(1, 137472, C, K, dil, mode, v) == 0, lib.ev_last_error()
    pl = dict(zip("MT KBG a_stages b_stages ntw acc smem tiles R rows1_pad rows2_pad".split(), list(v)))
    cpg = 8 if mode == 2 else 4
    n_cb = -(-C // (cpg * pl["KBG"]))
    for seed in range(5):
        sim_pair_overlap(seed, random.Random(seed).randint(1, 5), n_cb, K, pl["a_stages"], pl["b_stages"], n_chunks=C // 8)


def test_cross_tile_order_grouped():
    """Grouped launch: consecutive tiles of a CTA belong to layers with different taps, so c1(i + 1) may have fewer or more taps
    than epi2(i) has chunks."""
    for seed in range(30):
        rng = random.Random(seed)
        n = rng.randint(1, 6)
        sim_pair_overlap(seed, n, rng.randint(1, 3), [rng.choice((3, 7, 11)) for _ in range(n)], rng.randint(2, 4), rng.randint(2, 8),
                         n_chunks=rng.choice((4, 8, 16)))


def test_model_catches_xt_rewritten_under_the_other_warpgroups_c2():
    """Without the barrier ahead of epi1, a warp that has finished its own c2(i) and c1(i + 1) rewrites its xt rows while the other
    warpgroup's c2(i) still reads them: the model must see the wrong tile in the slot."""
    with pytest.raises(AssertionError):
        for seed in range(60):
            sim_pair_overlap(seed, 4, 1, 3, 4, 8, xt_barrier=False)
