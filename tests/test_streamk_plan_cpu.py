"""Pure-Python model of the stream-K decomposition arithmetic in csrc/decode_gemm_tc5.cu (skinny_tc5_kernel): which CTA
contributes to which feature tile, which partial tile it publishes to its one scratch slot, and which CTAs the reducing CTA
reads -- the invariants the deterministic fixed-order reduction relies on."""
import math

import pytest

BM, BK = 128, 64


def plan(N, K, n_sms=148):
    tiles, KB = math.ceil(N / BM), math.ceil(K / BK)
    units = tiles * KB
    grid = min(units, n_sms)
    chunk = math.ceil(units / grid)
    grid = math.ceil(units / chunk)
    return tiles, KB, units, chunk, grid


def segments(c, KB, units, chunk):
    """(tile, k_lo, k_hi, whole) for every segment CTA c processes, in order (mirrors the epilogue loop)."""
    u_lo, u_hi = c * chunk, min(units, (c + 1) * chunk)
    u, out = u_lo, []
    while u < u_hi:
        tile = u // KB
        seg_end = min(u_hi, (tile + 1) * KB)
        whole = (u == tile * KB) and (seg_end == (tile + 1) * KB)
        out.append((tile, u - tile * KB, seg_end - tile * KB, whole))
        u = seg_end
    return out


@pytest.mark.parametrize("N,K", [(6144, 2560), (2560, 4096), (19456, 2560), (2560, 9728), (151936, 2560),      # Qwen3-4B
                                 (4096, 2048), (2048, 2048), (12288, 2048), (2048, 6144),                       # Qwen3-1.7B
                                 (1024, 256), (256, 512), (1536, 512), (16, 64), (128, 8), (272, 136)])
@pytest.mark.parametrize("n_sms", [148, 132, 7])
def test_streamk_invariants(N, K, n_sms):
    tiles, KB, units, chunk, grid = plan(N, K, n_sms)
    assert grid <= n_sms and (grid - 1) * chunk < units <= grid * chunk          # every CTA has work, all units covered
    covered = {}
    for c in range(grid):
        segs = segments(c, KB, units, chunk)
        for i, (tile, lo, hi, whole) in enumerate(segs):
            if not whole:
                first_c = (tile * KB) // chunk
                if c == first_c:
                    assert i == len(segs) - 1                                    # the reducer meets the tile as its last segment
                else:                                                            # a publisher's partial starts its chunk:
                    assert i == 0                                                # one scratch slot per CTA suffices
            covered.setdefault(tile, []).append((lo, hi, c, whole))
    assert sorted(covered) == list(range(tiles))
    for tile, parts in covered.items():
        parts.sort()
        assert parts[0][0] == 0 and parts[-1][1] == KB and all(a[1] == b[0] for a, b in zip(parts, parts[1:]))   # k range tiled exactly once
        first_c, last_c = (tile * KB) // chunk, ((tile + 1) * KB - 1) // chunk    # what the reducing CTA computes
        assert [p[2] for p in parts] == list(range(first_c, last_c + 1))          # contributors = a contiguous CTA range, ascending k
        if len(parts) == 1:
            assert parts[0][3]                                                    # single owner -> direct epilogue, no scratch
        else:
            assert not any(p[3] for p in parts)
        # arrival counter: the last arriver sees (contributors - 1)
        assert last_c - first_c == len(parts) - 1
