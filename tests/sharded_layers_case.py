"""Host-side restatement of the render layers of the fused Gaussian-sharded step (tests/test_sharded_layers_*.py).

Layer membership travels with the record (include/sgr.h, SgrShardedLayer): owner s's block b of 256 Gaussians sends, to every rank d
its destination masks name, the layer byte of each such Gaussian (bit k = its local row lies in layer k's [begin, end)) into slots
s chunk + 256 b + 0, 1, ... of d's mask section, in ascending order, exactly where the record goes."""
from __future__ import annotations

import torch


def layer_bits(P_r, ranges):
    """Layer byte of every real Gaussian, rank-major: ranges[r] = [(begin, end) per layer] in rank r's local rows."""
    out = []
    for r, P in enumerate(P_r):
        bits = torch.zeros(P, dtype=torch.int64)
        for k, (b, e) in enumerate(ranges[r]):
            bits[b:e] |= 1 << k
        out.append(bits)
    return torch.cat(out) if out else torch.zeros(0, dtype=torch.int64)


def mask_slots(masks, P_r, chunk, world, ranges):
    """Per destination d: (slots of d's mask section, global ids, layer bytes) of the Gaussians delivered to d (the block runs)."""
    bits = layer_bits(P_r, ranges)
    offs = [sum(P_r[:r]) for r in range(world)]
    out = []
    for d in range(world):
        slots, gids = [], []
        for s in range(world):
            for b0 in range(0, P_r[s], 256):
                g = torch.arange(offs[s] + b0, offs[s] + min(P_r[s], b0 + 256))
                g = g[((masks[g] >> d) & 1).bool()]
                slots.append(s * chunk + b0 + torch.arange(g.numel()))
                gids.append(g)
        gids = torch.cat(gids) if gids else torch.zeros(0, dtype=torch.int64)
        out.append((torch.cat(slots) if slots else torch.zeros(0, dtype=torch.int64), gids, bits[gids]))
    return out


def layer_rows(P_r, ranges, k):
    """Global ids (rank-major) of layer k's rows: the rank-major concatenation of every rank's [begin, end)."""
    offs = [sum(P_r[:r]) for r in range(len(P_r))]
    return torch.cat([torch.arange(offs[r] + ranges[r][k][0], offs[r] + ranges[r][k][1]) for r in range(len(P_r))])


def case_ranges(P_r):
    """Two layers per rank: a background-like head and an objects-like tail.  Rank 0's head is empty, rank 1's tail covers its whole
    rows, the last rank's tail ends at its last real row (its slots past it are padding), every other tail starts 40 rows before the end."""
    out = []
    for r, P in enumerate(P_r):
        head = (0, 0) if r == 0 else (0, min(P, 97 + 13 * r))
        tail = (0, P) if r == 1 else (max(0, P - 40), P)
        out.append([head, tail])
    return out
