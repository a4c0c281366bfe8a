"""GPU: the hand-written onesweep radix sort of the binning stage against torch's stable sort (bit-exact, stable)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("n,nbits", [(1, 1), (31, 5), (257, 9), (3072, 12), (3073, 12), (100_003, 18), (1_000_000, 12),
                                     (2_500_000, 18), (700_001, 27), (50_000, 32),
                                     (6144, 10),   # a 1-bit last pass
                                     (9216, 19),   # three passes: the result lands in the other buffer
                                     (3071, 32), (2, 1),
                                     (5000, -18)])  # nbits < 0: every key equal, sorted over |nbits| bits
def test_sort_pairs_matches_stable_sort(n, nbits):
    from humangaussian_b200.rasterizer import device_sort_pairs
    equal = nbits < 0
    nbits = abs(nbits)
    g = torch.Generator(device="cpu").manual_seed(n + nbits)
    hi = (1 << nbits) if nbits < 31 else (1 << 31) - 1
    keys = torch.randint(0, hi, (n,), generator=g, dtype=torch.int64)
    if nbits == 32:  # exercise the top bit too
        keys = keys | (torch.randint(0, 2, (n,), generator=g, dtype=torch.int64) << 31)
    if n > 1000:     # heavy duplicates + a few empty digits, like tile ids
        keys[: n // 3] = keys[: n // 3] % 7
    if equal:
        keys[:] = (1 << nbits) - 1 - 5 * 512
    vals = torch.arange(n, dtype=torch.int64)
    k32 = keys.to(torch.int64).numpy().astype(np.uint32).view(np.int32)
    ks, vs = device_sort_pairs(torch.tensor(k32, device=DEV), vals.to(torch.int32).to(DEV), nbits)
    order = torch.sort(keys, stable=True).indices
    assert torch.equal(vs.cpu().to(torch.int64), vals[order]), "values are not in stable sorted order"
    assert np.array_equal(ks.cpu().numpy().view(np.uint32), keys[order].numpy().astype(np.uint32))


def test_sort_ignores_bits_above_nbits():
    from humangaussian_b200.rasterizer import device_sort_pairs
    n = 10_000
    g = torch.Generator().manual_seed(0)
    keys = torch.randint(0, 1 << 20, (n,), generator=g, dtype=torch.int64)
    ks, vs = device_sort_pairs(keys.to(torch.int32).to(DEV), torch.arange(n, dtype=torch.int32, device=DEV), 9)
    order = torch.sort(keys & 511, stable=True).indices
    assert torch.equal(vs.cpu().to(torch.int64), order)
