"""Host-side restatement of the paired shared-memory layout of the forward recurrence (csrc/rnn_core.cuh
`paired_index`, used by `dots_chunk2b` / `allgather_units<..., PAIRED>`), checked for the properties the kernels rely on.
No GPU needed: the CUDA side is covered by the parity tests; this pins the index algebra for every config that uses it.
"""
import itertools

import pytest


def paired_index(j: int, b: int, KL: int, BS: int) -> int:
    CW = 4 * KL
    return ((((j // CW) * 4 + (j & 3)) * (BS // 2) + (b >> 1)) * KL + (j % CW) // 4) * 2 + (b & 1)


# (H, KL, UPL, BS) of the forward configs dispatched with the batch-paired form (csrc/rnn_rec.cu plan_rec_fwd)
CONFIGS = [(256, 16, 4, 4)]


@pytest.mark.parametrize("H,KL,UPL,BS", CONFIGS)
def test_paired_layout_is_a_permutation_of_the_state_buffer(H, KL, UPL, BS):
    idx = sorted(paired_index(j, b, KL, BS) for j in range(H) for b in range(BS))
    assert idx == list(range(H * BS))       # same footprint as the [BS][H] layout: the double buffer size is unchanged


@pytest.mark.parametrize("H,KL,UPL,BS", CONFIGS)
def test_reader_words_are_aligned_pairs_and_conflict_free(H, KL, UPL, BS):
    NP = BS // 2
    for ca, e, am in itertools.product(range(H // (4 * KL)), range(4), range(NP)):
        words = []
        for kl in range(KL):
            k = ca * 4 * KL + kl * 4 + e
            qh = (kl & (BS - 1)) >> 1              # lanes of one LDS.64 read different pair slots (am ^ qh)
            first = paired_index(k, 2 * (am ^ qh), KL, BS)
            assert first % 2 == 0 and paired_index(k, 2 * (am ^ qh) + 1, KL, BS) == first + 1   # one 8-byte word
            # address the kernel computes: (((ca*4 + e)*NP + (am ^ qh))*KL + kl)*2
            assert first == (((ca * 4 + e) * NP + (am ^ qh)) * KL + kl) * 2
            words.append(first)
        banks = [(w % 32) for w in words]           # 4-byte banks of the first float of every 8-byte word
        assert len(set(banks)) == KL                # the KL k-lanes hit KL distinct bank pairs


@pytest.mark.parametrize("H,KL,UPL,BS", CONFIGS)
def test_exchange_stores_are_16_byte_groups(H, KL, UPL, BS):
    """One st.async carries units j and j+4 (j % 8 < 4) for the two batch rows of a pair: four consecutive floats."""
    UPW = (32 // KL) * UPL
    assert UPW % 8 == 0
    for col0 in range(0, H, UPW):
        for ue, pr in itertools.product(range(UPW // 2), range(BS // 2)):
            u = (ue // 4) * 8 + (ue % 4)
            j = col0 + u
            base = paired_index(j, 2 * pr, KL, BS)
            assert base % 4 == 0
            assert [paired_index(j, 2 * pr + 1, KL, BS), paired_index(j + 4, 2 * pr, KL, BS),
                    paired_index(j + 4, 2 * pr + 1, KL, BS)] == [base + 1, base + 2, base + 3]
    # every (unit, batch) of a warp is covered exactly once
    seen = set()
    for ue, pr in itertools.product(range(UPW // 2), range(BS // 2)):
        u = (ue // 4) * 8 + (ue % 4)
        seen |= {(u, 2 * pr), (u, 2 * pr + 1), (u + 4, 2 * pr), (u + 4, 2 * pr + 1)}
    assert seen == {(u, b) for u in range(UPW) for b in range(BS)}
