"""Host-side split of a submap over ranks (SURVEY.md 8e): the mirror of owner_of() in csrc/mapping.cu.

Cells are cubes of edge CELL = 1 m * (1 + 1e-5) (float32), slab = 8 cells along x, owner(slab) = slab mod world.
A rank's shard = every map point whose cell_x lies in one of its slabs or within ONE cell of one (the halo), so the
27-cell neighbourhood of any query the rank owns is complete and its 5-NN equals the global 5-NN whenever the
reference would accept it (5th distance < 1 m)."""
import numpy as np

CELL = np.float32(1.0) * (np.float32(1.0) + np.float32(1e-5))
INV_CELL = np.float32(1.0) / CELL
SLAB = 8


def cell_x(x):
    return np.floor(np.asarray(x, np.float32) * INV_CELL).astype(np.int64)


def owner_of_cell(cx, world):
    """floor division and a non-negative remainder (Python semantics), as owner_of() on the device for every cell"""
    return ((np.asarray(cx, np.int64) + (1 << 20)) // SLAB) % world


def shard_mask(cloud, rank, world):
    """boolean mask of the points of `cloud` (n, >=3) that belong to `rank`'s shard (owned slabs + one-cell halo)"""
    if world == 1:
        return np.ones(len(cloud), bool)
    cx = cell_x(cloud[:, 0])
    return (owner_of_cell(cx, world) == rank) | (owner_of_cell(cx - 1, world) == rank) | (owner_of_cell(cx + 1, world) == rank)


def shard_cloud(cloud, rank, world):
    return np.ascontiguousarray(cloud[shard_mask(cloud, rank, world)])
