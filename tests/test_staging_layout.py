"""Host-side model of the shared-memory layout of the staged activation vector (calm_b200/csrc/common.cuh: xs_index,
xs_swz, xs_aux_floats).  The kernels' parity tests prove the values; this file pins the two properties the layout exists
for -- the staging stores and the matvec loads are both free of shared-memory bank conflicts -- so that a later change of
the permutation cannot silently bring back the 4-way (fp8) / 8-way (gf4) store conflicts of the unswizzled layout."""
import numpy as np
import pytest

VW = {16: 8, 8: 16, 4: 32}  # weights per 16-byte vector (common.cuh WFmt)


def xs_swz(dbits, q):
    return (q * (8 // (VW[dbits] // 4))) & 31


def xs_index(dbits, j):
    vw = VW[dbits]
    quads = vw // 4
    v, w = divmod(j, vw)
    c, lane = v >> 5, v & 31
    q = w >> 2
    return (((c * quads + q) << 5) + (lane ^ xs_swz(dbits, q))) * 4 + (w & 3)


def xs_floats(dbits, n):
    nvec = n // VW[dbits]
    return ((nvec + 31) & ~31) * VW[dbits]


def bank_groups(float_offsets):
    """16-byte bank group (0..7) of each 16-byte access, given its first float's offset."""
    return [(off // 4) % 8 for off in float_offsets]


@pytest.mark.parametrize("dbits", [16, 8, 4])
@pytest.mark.parametrize("n", [256, 4096, 14336])
def test_layout_is_a_permutation_of_the_padded_vector(dbits, n):
    total = xs_floats(dbits, n)
    slots = np.array([xs_index(dbits, j) for j in range(total)])
    assert slots.min() == 0 and slots.max() == total - 1
    assert len(np.unique(slots)) == total
    # four consecutive activations stay one aligned float4 (the staging writes and the matvec reads are 16-byte accesses)
    for j in range(0, total, 4):
        assert slots[j] % 4 == 0 and list(slots[j:j + 4]) == list(range(slots[j], slots[j] + 4))


@pytest.mark.parametrize("dbits", [16, 8, 4])
@pytest.mark.parametrize("nthr", [256, 384, 512])
def test_staging_stores_are_conflict_free(dbits, nthr):
    """stage_vector_batched: thread t stores the float4 i = t + k * nthr of x to xs_index(4 i).  A 16-byte store is
    issued in phases of 8 consecutive lanes: the 8 stores of a phase must fall in 8 different 16-byte bank groups."""
    n = 14336
    for k in range(2):
        for warp in range(nthr // 32):
            for phase in range(4):
                lanes = range(warp * 32 + phase * 8, warp * 32 + phase * 8 + 8)
                offs = [xs_index(dbits, 4 * (t + k * nthr)) for t in lanes if 4 * (t + k * nthr) < n]
                groups = bank_groups(offs)
                assert len(set(groups)) == len(groups), (dbits, nthr, k, warp, phase, groups)


@pytest.mark.parametrize("dbits", [16, 8, 4])
def test_matvec_loads_read_the_lane_s_own_quads_without_conflicts(dbits):
    """rows_consume / RingWarp::consume_all: lane l of a warp reads quad q of its vector v = 32 c + l at float4 index
    (c Q + q) 32 + (l ^ xs_swz(q)): the activations 4 q .. 4 q + 3 of that vector, 32 distinct slots of one 512-byte line."""
    vw = VW[dbits]
    quads = vw // 4
    for c in range(3):
        for q in range(quads):
            offs = []
            for lane in range(32):
                f4 = (c * quads + q) * 32 + (lane ^ xs_swz(dbits, q))
                v = 32 * c + lane
                assert f4 * 4 == xs_index(dbits, v * vw + 4 * q)
                offs.append(f4 * 4)
            assert sorted(offs) == list(range(min(offs), min(offs) + 128, 4))  # one contiguous 512-byte line, every slot once
            for phase in range(4):
                groups = bank_groups(offs[phase * 8:phase * 8 + 8])
                assert len(set(groups)) == 8


def test_gf4_group_sums_sit_behind_the_vector_in_plain_order():
    """xs_aux_floats: group g (activations 8 g .. 8 g + 7, one gf4 word) is float xs_floats(n) + g; lane l of chunk c reads
    its vector's four sums as the float4 at index 32 c + l behind the vector -- the groups 4 v .. 4 v + 3 of vector v."""
    n = 4096
    base = xs_floats(4, n)
    assert base % 4 == 0
    for v in (0, 1, 31, 32, 127):
        groups = [4 * v + k for k in range(4)]
        assert [base + g for g in groups] == list(range(base + 4 * v, base + 4 * v + 4))
        assert all(8 * g // VW[4] == v for g in groups)  # each of those groups belongs to vector v
