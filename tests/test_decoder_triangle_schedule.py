"""The work units of the decoder's triangle sweep (gae_tri_tc_kernel, csrc/gae_tc.cu), restated in Python.

CTA (x, y) takes 128-row block I = x and the y-th of `splits` step ranges of its J tiles: the 64-column tiles from block I's
own diagonal block to the last tile holding a column j < n.  A tile inside the diagonal block counts its logits once (it holds
both orders of each pair); a tile above it counts them for (i, j) and (j, i).  Over all CTAs every ordered pair of 64-row
groups must then be counted exactly once, for any split count, and the launch order (x ascending) must hand out the longest
units first so that the SMs finish close to together."""
import heapq

import pytest

BT, JW = 128, 64


def tri_ctas(n, splits):
    """(block, J tile range) of every non-empty CTA, in launch order, as launch_sweep / decoder_sweep compute them"""
    nb, n_jt = -(-n // BT), -(-n // JW)
    splits = max(1, min(splits, n_jt))
    out = []
    for y in range(splits):
        for blk in range(nb):
            first = blk * BT // JW
            per = -(-(n_jt - first) // splits)
            jt0 = first + y * per
            jt1 = min(n_jt, jt0 + per)
            if jt0 < jt1:
                out.append((blk, range(jt0, jt1)))
    return out


@pytest.mark.parametrize("n", [100, 128, 129, 255, 256, 1281, 2049, 8200])
@pytest.mark.parametrize("splits", [1, 2, 3, 7, 40, 1000])
def test_triangle_counts_every_pair_once(n, splits):
    n_jt = -(-n // JW)
    count = [[0] * n_jt for _ in range(n_jt)]          # 64-row group a against 64-column tile b
    seen = set()
    for blk, tiles in tri_ctas(n, splits):
        for t in tiles:
            assert (blk, t) not in seen
            seen.add((blk, t))
            for a in (2 * blk, 2 * blk + 1):
                if a >= n_jt:
                    continue                           # rows past n: masked in the kernel
                count[a][t] += 1
                if t // 2 != blk:
                    count[t][a] += 1                   # dZ_J and the doubled loss stand for the mirror tile
    assert all(c == 1 for row in count for c in row)


@pytest.mark.parametrize("n,splits", [(8200, 7), (2049, 3), (100_000, 2)])
def test_triangle_step_ranges_are_even(n, splits):
    """Within a block, the step ranges differ by at most one tile, apart from the last one (what is left)."""
    by_block = {}
    for blk, tiles in tri_ctas(n, splits):
        by_block.setdefault(blk, []).append(len(tiles))
    for lens in by_block.values():
        assert max(lens[:-1] or lens) - min(lens[:-1] or lens) <= 1 and lens[-1] <= max(lens)


@pytest.mark.parametrize("n", [1_000_000, 250_000])
def test_triangle_longest_first_fills_the_machine(n, sms=132):
    """Blocks launch in order of decreasing work; greedy assignment to 132 SMs (the block scheduler) ends within 1 % of the
    ideal, total work / SMs."""
    ctas = tri_ctas(n, -(-sms // -(-n // BT)))         # automatic split count: fill one wave
    lens = [len(t) for _, t in ctas]
    assert lens == sorted(lens, reverse=True)
    free = [0] * sms
    for w in lens:
        heapq.heappush(free, heapq.heappop(free) + w)
    ideal = sum(lens) / sms
    assert max(free) <= 1.01 * ideal, (max(free), ideal)
