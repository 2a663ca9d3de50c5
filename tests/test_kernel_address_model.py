"""CPU restatement of the shared-memory addressing of the histogram kernels (csrc/hist_common.cuh::accumulate_row,
hist_kernel.cu::full_pass with one or two feature groups per CTA): at every step the 32 lanes of a warp must address
32 different banks for ANY bin values (one wavefront per red.shared.add), and every (row, feature) pair must be added
exactly once to the cell of its (bin, plane, feature slot).  The GPU suite proves the sums; this pins the bank layout the
design (DESIGN.md 4.1) rests on: one wavefront per shared atomic instruction."""
import numpy as np
import pytest

GROUP_BYTES = 65536          # int32 [256 bins][2 planes][32 slots]


def bank(addr):
    return (addr >> 2) & 31


def full_pass_lanes(groups_per_cta):
    """lane -> (row of the warp step, group of the CTA, 16-byte half, rotation): hist_kernel.cu::full_pass"""
    lanes_per_row = 2 * groups_per_cta
    out = []
    for lane in range(32):
        sub, gsel, half = lane // lanes_per_row, (lane % lanes_per_row) >> 1, lane & 1
        out.append((sub, gsel, half, sub * groups_per_cta + gsel))
    return out


@pytest.mark.parametrize("groups_per_cta", [1, 2])
def test_full_groups_are_bank_conflict_free_and_complete(groups_per_cta):
    rng = np.random.RandomState(groups_per_cta)
    lanes = full_pass_lanes(groups_per_cta)
    rows_per_warp = 32 // (2 * groups_per_cta)
    bins = rng.randint(0, 256, size=(rows_per_warp, groups_per_cta, 32))     # [row][group][feature slot]
    seen = set()
    for j in range(16):
        banks = []
        for sub, gsel, half, rot in lanes:
            slot = half * 16 + ((j + rot) & 15)                 # rotate_bytes: step j reads source byte (j + rot) & 15
            b = int(bins[sub, gsel, slot])
            addr = gsel * GROUP_BYTES + half * 64 + b * 256 + ((j + rot) & 15) * 4
            assert addr == gsel * GROUP_BYTES + b * 256 + slot * 4          # cell [bin][plane 0][slot]
            banks.append(bank(addr))
            seen.add((sub, gsel, slot))
        assert len(set(banks)) == 32, (j, sorted(banks))
        assert len({bank(a + 128) for a in banks}) <= 32                    # the h plane is 128 B further: same banks, next instruction
    assert len(seen) == rows_per_warp * groups_per_cta * 32                # every (row, group, feature) exactly once
