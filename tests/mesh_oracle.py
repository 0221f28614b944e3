"""numpy restatement of the marching-cubes stages of localrf_b200/csrc/lrf_mesh.cu (lrf_mesh_cells, lrf_mesh_extract),
applied to given lattice values, and a float64 restatement of the scalar field A that lrf_mesh_lattice samples.
TEST INFRASTRUCTURE: nothing under localrf_b200/ imports it.

The cells and extract stages are restated bit for bit: the same fp32 round-to-nearest vertex arithmetic, the same edge
and triangle keys, the same sort orders.  This file keeps its own copy of the 256-case triangle table.  cells_np /
extract_np restate the same stages with array operations, for lattices of up to ~10^7 cells; owner32 restates the
owner rule in float32 and probe_slots the edge table's occupied slots."""
import numpy as np
import torch
import torch.nn.functional as Fn

# corner c of a cell sits at (c & 1 ^ (c >> 1) & 1, (c >> 1) & 1, (c >> 2) & 1): 0 (0,0,0), 1 (1,0,0), 2 (1,1,0),
# 3 (0,1,0), then the same four at z = 1
CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
# the twelve edges as (corner, corner)
EDGES = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]

# The widely published 256-case triangle table: row i lists the edges of the triangles of the case whose corner c is
# inside when bit c of i is set, three edges per triangle.
TRI_TABLE = [
    [], [0, 8, 3], [0, 1, 9], [1, 8, 3, 9, 8, 1], [1, 2, 10], [0, 8, 3, 1, 2, 10], [9, 2, 10, 0, 2, 9],
    [2, 8, 3, 2, 10, 8, 10, 9, 8], [3, 11, 2], [0, 11, 2, 8, 11, 0], [1, 9, 0, 2, 3, 11],
    [1, 11, 2, 1, 9, 11, 9, 8, 11], [3, 10, 1, 11, 10, 3], [0, 10, 1, 0, 8, 10, 8, 11, 10],
    [3, 9, 0, 3, 11, 9, 11, 10, 9], [9, 8, 10, 10, 8, 11], [4, 7, 8], [4, 3, 0, 7, 3, 4], [0, 1, 9, 8, 4, 7],
    [4, 1, 9, 4, 7, 1, 7, 3, 1], [1, 2, 10, 8, 4, 7], [3, 4, 7, 3, 0, 4, 1, 2, 10], [9, 2, 10, 9, 0, 2, 8, 4, 7],
    [2, 10, 9, 2, 9, 7, 2, 7, 3, 7, 9, 4], [8, 4, 7, 3, 11, 2], [11, 4, 7, 11, 2, 4, 2, 0, 4],
    [9, 0, 1, 8, 4, 7, 2, 3, 11], [4, 7, 11, 9, 4, 11, 9, 11, 2, 9, 2, 1], [3, 10, 1, 3, 11, 10, 7, 8, 4],
    [1, 11, 10, 1, 4, 11, 1, 0, 4, 7, 11, 4], [4, 7, 8, 9, 0, 11, 9, 11, 10, 11, 0, 3],
    [4, 7, 11, 4, 11, 9, 9, 11, 10], [9, 5, 4], [9, 5, 4, 0, 8, 3], [0, 5, 4, 1, 5, 0], [8, 5, 4, 8, 3, 5, 3, 1, 5],
    [1, 2, 10, 9, 5, 4], [3, 0, 8, 1, 2, 10, 4, 9, 5], [5, 2, 10, 5, 4, 2, 4, 0, 2],
    [2, 10, 5, 3, 2, 5, 3, 5, 4, 3, 4, 8], [9, 5, 4, 2, 3, 11], [0, 11, 2, 0, 8, 11, 4, 9, 5],
    [0, 5, 4, 0, 1, 5, 2, 3, 11], [2, 1, 5, 2, 5, 8, 2, 8, 11, 4, 8, 5], [10, 3, 11, 10, 1, 3, 9, 5, 4],
    [4, 9, 5, 0, 8, 1, 8, 10, 1, 8, 11, 10], [5, 4, 0, 5, 0, 11, 5, 11, 10, 11, 0, 3],
    [5, 4, 8, 5, 8, 10, 10, 8, 11], [9, 7, 8, 5, 7, 9], [9, 3, 0, 9, 5, 3, 5, 7, 3], [0, 7, 8, 0, 1, 7, 1, 5, 7],
    [1, 5, 3, 3, 5, 7], [9, 7, 8, 9, 5, 7, 10, 1, 2], [10, 1, 2, 9, 5, 0, 5, 3, 0, 5, 7, 3],
    [8, 0, 2, 8, 2, 5, 8, 5, 7, 10, 5, 2], [2, 10, 5, 2, 5, 3, 3, 5, 7], [7, 9, 5, 7, 8, 9, 3, 11, 2],
    [9, 5, 7, 9, 7, 2, 9, 2, 0, 2, 7, 11], [2, 3, 11, 0, 1, 8, 1, 7, 8, 1, 5, 7], [11, 2, 1, 11, 1, 7, 7, 1, 5],
    [9, 5, 8, 8, 5, 7, 10, 1, 3, 10, 3, 11], [5, 7, 0, 5, 0, 9, 7, 11, 0, 1, 0, 10, 11, 10, 0],
    [11, 10, 0, 11, 0, 3, 10, 5, 0, 8, 0, 7, 5, 7, 0], [11, 10, 5, 7, 11, 5], [10, 6, 5], [0, 8, 3, 5, 10, 6],
    [9, 0, 1, 5, 10, 6], [1, 8, 3, 1, 9, 8, 5, 10, 6], [1, 6, 5, 2, 6, 1], [1, 6, 5, 1, 2, 6, 3, 0, 8],
    [9, 6, 5, 9, 0, 6, 0, 2, 6], [5, 9, 8, 5, 8, 2, 5, 2, 6, 3, 2, 8], [2, 3, 11, 10, 6, 5],
    [11, 0, 8, 11, 2, 0, 10, 6, 5], [0, 1, 9, 2, 3, 11, 5, 10, 6], [5, 10, 6, 1, 9, 2, 9, 11, 2, 9, 8, 11],
    [6, 3, 11, 6, 5, 3, 5, 1, 3], [0, 8, 11, 0, 11, 5, 0, 5, 1, 5, 11, 6], [3, 11, 6, 0, 3, 6, 0, 6, 5, 0, 5, 9],
    [6, 5, 9, 6, 9, 11, 11, 9, 8], [5, 10, 6, 4, 7, 8], [4, 3, 0, 4, 7, 3, 6, 5, 10], [1, 9, 0, 5, 10, 6, 8, 4, 7],
    [10, 6, 5, 1, 9, 7, 1, 7, 3, 7, 9, 4], [6, 1, 2, 6, 5, 1, 4, 7, 8], [1, 2, 5, 5, 2, 6, 3, 0, 4, 3, 4, 7],
    [8, 4, 7, 9, 0, 5, 0, 6, 5, 0, 2, 6], [7, 3, 9, 7, 9, 4, 3, 2, 9, 5, 9, 6, 2, 6, 9],
    [3, 11, 2, 7, 8, 4, 10, 6, 5], [5, 10, 6, 4, 7, 2, 4, 2, 0, 2, 7, 11],
    [0, 1, 9, 4, 7, 8, 2, 3, 11, 5, 10, 6], [9, 2, 1, 9, 11, 2, 9, 4, 11, 7, 11, 4, 5, 10, 6],
    [8, 4, 7, 3, 11, 5, 3, 5, 1, 5, 11, 6], [5, 1, 11, 5, 11, 6, 1, 0, 11, 7, 11, 4, 0, 4, 11],
    [0, 5, 9, 0, 6, 5, 0, 3, 6, 11, 6, 3, 8, 4, 7], [6, 5, 9, 6, 9, 11, 4, 7, 9, 7, 11, 9], [10, 4, 9, 6, 4, 10],
    [4, 10, 6, 4, 9, 10, 0, 8, 3], [10, 0, 1, 10, 6, 0, 6, 4, 0], [8, 3, 1, 8, 1, 6, 8, 6, 4, 6, 1, 10],
    [1, 4, 9, 1, 2, 4, 2, 6, 4], [3, 0, 8, 1, 2, 9, 2, 4, 9, 2, 6, 4], [0, 2, 4, 4, 2, 6],
    [8, 3, 2, 8, 2, 4, 4, 2, 6], [10, 4, 9, 10, 6, 4, 11, 2, 3], [0, 8, 2, 2, 8, 11, 4, 9, 10, 4, 10, 6],
    [3, 11, 2, 0, 1, 6, 0, 6, 4, 6, 1, 10], [6, 4, 1, 6, 1, 10, 4, 8, 1, 2, 1, 11, 8, 11, 1],
    [9, 6, 4, 9, 3, 6, 9, 1, 3, 11, 6, 3], [8, 11, 1, 8, 1, 0, 11, 6, 1, 9, 1, 4, 6, 4, 1],
    [3, 11, 6, 3, 6, 0, 0, 6, 4], [6, 4, 8, 11, 6, 8], [7, 10, 6, 7, 8, 10, 8, 9, 10],
    [0, 7, 3, 0, 10, 7, 0, 9, 10, 6, 7, 10], [10, 6, 7, 1, 10, 7, 1, 7, 8, 1, 8, 0],
    [10, 6, 7, 10, 7, 1, 1, 7, 3], [1, 2, 6, 1, 6, 8, 1, 8, 9, 8, 6, 7],
    [2, 6, 9, 2, 9, 1, 6, 7, 9, 0, 9, 3, 7, 3, 9], [7, 8, 0, 7, 0, 6, 6, 0, 2], [7, 3, 2, 6, 7, 2],
    [2, 3, 11, 10, 6, 8, 10, 8, 9, 8, 6, 7], [2, 0, 7, 2, 7, 11, 0, 9, 7, 6, 7, 10, 9, 10, 7],
    [1, 8, 0, 1, 7, 8, 1, 10, 7, 6, 7, 10, 2, 3, 11], [11, 2, 1, 11, 1, 7, 10, 6, 1, 6, 7, 1],
    [8, 9, 6, 8, 6, 7, 9, 1, 6, 11, 6, 3, 1, 3, 6], [0, 9, 1, 11, 6, 7], [7, 8, 0, 7, 0, 6, 3, 11, 0, 11, 6, 0],
    [7, 11, 6], [7, 6, 11], [3, 0, 8, 11, 7, 6], [0, 1, 9, 11, 7, 6], [8, 1, 9, 8, 3, 1, 11, 7, 6],
    [10, 1, 2, 6, 11, 7], [1, 2, 10, 3, 0, 8, 6, 11, 7], [2, 9, 0, 2, 10, 9, 6, 11, 7],
    [6, 11, 7, 2, 10, 3, 10, 8, 3, 10, 9, 8], [7, 2, 3, 6, 2, 7], [7, 0, 8, 7, 6, 0, 6, 2, 0],
    [2, 7, 6, 2, 3, 7, 0, 1, 9], [1, 6, 2, 1, 8, 6, 1, 9, 8, 8, 7, 6], [10, 7, 6, 10, 1, 7, 1, 3, 7],
    [10, 7, 6, 1, 7, 10, 1, 8, 7, 1, 0, 8], [0, 3, 7, 0, 7, 10, 0, 10, 9, 6, 10, 7],
    [7, 6, 10, 7, 10, 8, 8, 10, 9], [6, 8, 4, 11, 8, 6], [3, 6, 11, 3, 0, 6, 0, 4, 6],
    [8, 6, 11, 8, 4, 6, 9, 0, 1], [9, 4, 6, 9, 6, 3, 9, 3, 1, 11, 3, 6], [6, 8, 4, 6, 11, 8, 2, 10, 1],
    [1, 2, 10, 3, 0, 11, 0, 6, 11, 0, 4, 6], [4, 11, 8, 4, 6, 11, 0, 2, 9, 2, 10, 9],
    [10, 9, 3, 10, 3, 2, 9, 4, 3, 11, 3, 6, 4, 6, 3], [8, 2, 3, 8, 4, 2, 4, 6, 2], [0, 4, 2, 4, 6, 2],
    [1, 9, 0, 2, 3, 4, 2, 4, 6, 4, 3, 8], [1, 9, 4, 1, 4, 2, 2, 4, 6], [8, 1, 3, 8, 6, 1, 8, 4, 6, 6, 10, 1],
    [10, 1, 0, 10, 0, 6, 6, 0, 4], [4, 6, 3, 4, 3, 8, 6, 10, 3, 0, 3, 9, 10, 9, 3], [10, 9, 4, 6, 10, 4],
    [4, 9, 5, 7, 6, 11], [0, 8, 3, 4, 9, 5, 11, 7, 6], [5, 0, 1, 5, 4, 0, 7, 6, 11],
    [11, 7, 6, 8, 3, 4, 3, 5, 4, 3, 1, 5], [9, 5, 4, 10, 1, 2, 7, 6, 11], [6, 11, 7, 1, 2, 10, 0, 8, 3, 4, 9, 5],
    [7, 6, 11, 5, 4, 10, 4, 2, 10, 4, 0, 2], [3, 4, 8, 3, 5, 4, 3, 2, 5, 10, 5, 2, 11, 7, 6],
    [7, 2, 3, 7, 6, 2, 5, 4, 9], [9, 5, 4, 0, 8, 6, 0, 6, 2, 6, 8, 7], [3, 6, 2, 3, 7, 6, 1, 5, 0, 5, 4, 0],
    [6, 2, 8, 6, 8, 7, 2, 1, 8, 4, 8, 5, 1, 5, 8], [9, 5, 4, 10, 1, 6, 1, 7, 6, 1, 3, 7],
    [1, 6, 10, 1, 7, 6, 1, 0, 7, 8, 7, 0, 9, 5, 4], [4, 0, 10, 4, 10, 5, 0, 3, 10, 6, 10, 7, 3, 7, 10],
    [7, 6, 10, 7, 10, 8, 5, 4, 10, 4, 8, 10], [6, 9, 5, 6, 11, 9, 11, 8, 9], [3, 6, 11, 0, 6, 3, 0, 5, 6, 0, 9, 5],
    [0, 11, 8, 0, 5, 11, 0, 1, 5, 5, 6, 11], [6, 11, 3, 6, 3, 5, 5, 3, 1],
    [1, 2, 10, 9, 5, 11, 9, 11, 8, 11, 5, 6], [0, 11, 3, 0, 6, 11, 0, 9, 6, 5, 6, 9, 1, 2, 10],
    [11, 8, 5, 11, 5, 6, 8, 0, 5, 10, 5, 2, 0, 2, 5], [6, 11, 3, 6, 3, 5, 2, 10, 3, 10, 5, 3],
    [5, 8, 9, 5, 2, 8, 5, 6, 2, 3, 8, 2], [9, 5, 6, 9, 6, 0, 0, 6, 2],
    [1, 5, 8, 1, 8, 0, 5, 6, 8, 3, 8, 2, 6, 2, 8], [1, 5, 6, 2, 1, 6],
    [1, 3, 6, 1, 6, 10, 3, 8, 6, 5, 6, 9, 8, 9, 6], [10, 1, 0, 10, 0, 6, 9, 5, 0, 5, 6, 0], [0, 3, 8, 5, 6, 10],
    [10, 5, 6], [11, 5, 10, 7, 5, 11], [11, 5, 10, 11, 7, 5, 8, 3, 0], [5, 11, 7, 5, 10, 11, 1, 9, 0],
    [10, 7, 5, 10, 11, 7, 9, 8, 1, 8, 3, 1], [11, 1, 2, 11, 7, 1, 7, 5, 1], [0, 8, 3, 1, 2, 7, 1, 7, 5, 7, 2, 11],
    [9, 7, 5, 9, 2, 7, 9, 0, 2, 2, 11, 7], [7, 5, 2, 7, 2, 11, 5, 9, 2, 3, 2, 8, 9, 8, 2],
    [2, 5, 10, 2, 3, 5, 3, 7, 5], [8, 2, 0, 8, 5, 2, 8, 7, 5, 10, 2, 5], [9, 0, 1, 5, 10, 3, 5, 3, 7, 3, 10, 2],
    [9, 8, 2, 9, 2, 1, 8, 7, 2, 10, 2, 5, 7, 5, 2], [1, 3, 5, 3, 7, 5], [0, 8, 7, 0, 7, 1, 1, 7, 5],
    [9, 0, 3, 9, 3, 5, 5, 3, 7], [9, 8, 7, 5, 9, 7], [5, 8, 4, 5, 10, 8, 10, 11, 8],
    [5, 0, 4, 5, 11, 0, 5, 10, 11, 11, 3, 0], [0, 1, 9, 8, 4, 10, 8, 10, 11, 10, 4, 5],
    [10, 11, 4, 10, 4, 5, 11, 3, 4, 9, 4, 1, 3, 1, 4], [2, 5, 1, 2, 8, 5, 2, 11, 8, 4, 5, 8],
    [0, 4, 11, 0, 11, 3, 4, 5, 11, 2, 11, 1, 5, 1, 11], [0, 2, 5, 0, 5, 9, 2, 11, 5, 4, 5, 8, 11, 8, 5],
    [9, 4, 5, 2, 11, 3], [2, 5, 10, 3, 5, 2, 3, 4, 5, 3, 8, 4], [5, 10, 2, 5, 2, 4, 4, 2, 0],
    [3, 10, 2, 3, 5, 10, 3, 8, 5, 4, 5, 8, 0, 1, 9], [5, 10, 2, 5, 2, 4, 1, 9, 2, 9, 4, 2],
    [8, 4, 5, 8, 5, 3, 3, 5, 1], [0, 4, 5, 1, 0, 5], [8, 4, 5, 8, 5, 3, 9, 0, 5, 0, 3, 5], [9, 4, 5],
    [4, 11, 7, 4, 9, 11, 9, 10, 11], [0, 8, 3, 4, 9, 7, 9, 11, 7, 9, 10, 11], [1, 10, 11, 1, 11, 4, 1, 4, 0, 7, 4, 11],
    [3, 1, 4, 3, 4, 8, 1, 10, 4, 7, 4, 11, 10, 11, 4], [4, 11, 7, 9, 11, 4, 9, 2, 11, 9, 1, 2],
    [9, 7, 4, 9, 11, 7, 9, 1, 11, 2, 11, 1, 0, 8, 3], [11, 7, 4, 11, 4, 2, 2, 4, 0],
    [11, 7, 4, 11, 4, 2, 8, 3, 4, 3, 2, 4], [2, 9, 10, 2, 7, 9, 2, 3, 7, 7, 4, 9],
    [9, 10, 7, 9, 7, 4, 10, 2, 7, 8, 7, 0, 2, 0, 7], [3, 7, 10, 3, 10, 2, 7, 4, 10, 1, 10, 0, 4, 0, 10],
    [1, 10, 2, 8, 7, 4], [4, 9, 1, 4, 1, 7, 7, 1, 3], [4, 9, 1, 4, 1, 7, 0, 8, 1, 8, 7, 1], [4, 0, 3, 7, 4, 3],
    [4, 8, 7], [9, 10, 8, 10, 11, 8], [3, 0, 9, 3, 9, 11, 11, 9, 10], [0, 1, 10, 0, 10, 8, 8, 10, 11],
    [3, 1, 10, 11, 3, 10], [1, 2, 11, 1, 11, 9, 9, 11, 8], [3, 0, 9, 3, 9, 11, 1, 2, 9, 2, 11, 9],
    [0, 2, 11, 8, 0, 11], [3, 2, 11], [2, 3, 8, 2, 8, 10, 10, 8, 9], [9, 10, 2, 0, 9, 2],
    [2, 3, 8, 2, 8, 10, 0, 1, 8, 1, 10, 8], [1, 10, 2], [1, 3, 8, 9, 1, 8], [0, 9, 1], [0, 3, 8], [],
]
N_TRI = [len(r) // 3 for r in TRI_TABLE]
HALF = 1 << 19                     # lattice indices lie in [-2^19, 2^19) on every axis


def edge_key(i, axis):
    """The global key of the lattice edge from point i (its lower end) along `axis`: 20 bits per axis, then the axis."""
    return ((int(i[0]) + HALF) << 42) | ((int(i[1]) + HALF) << 22) | ((int(i[2]) + HALF) << 2) | int(axis)


def cell_key(c):
    """The 60-bit key of the cell whose lower corner is lattice point c."""
    return ((int(c[0]) + HALF) << 40) | ((int(c[1]) + HALF) << 20) | (int(c[2]) + HALF)


def lattice_coord(i, origin, voxel_size):
    """origin + i voxel_size per axis in fp32, round to nearest -> [3] float32."""
    return np.array([np.float32(origin[a]) + np.float32(int(i[a])) * np.float32(voxel_size) for a in range(3)],
                    np.float32)


def edge_vertex(i, axis, va, vb, level, origin, voxel_size):
    """The vertex of the edge from point i (value va) to point i + e_axis (value vb): t = (level - va) / (vb - va) in
    fp32, 0 when not finite, clamped to [0, 1]; the vertex moves from the lower point along the axis only."""
    pa = lattice_coord(i, origin, voxel_size)
    j = list(i)
    j[axis] += 1
    pb = lattice_coord(j, origin, voxel_size)
    with np.errstate(all="ignore"):
        t = (np.float32(level) - np.float32(va)) / (np.float32(vb) - np.float32(va))
    t = np.float32(0) if not np.isfinite(t) else np.float32(min(max(t, np.float32(0)), np.float32(1)))
    v = pa.copy()
    v[axis] = pa[axis] + t * (pb[axis] - pa[axis])
    return v


def case_index(v8, level):
    """Bit c set when corner c is inside (value >= level; NaN is outside)."""
    return sum(1 << c for c in range(8) if np.float32(v8[c]) >= np.float32(level))


def cells(values, lo, level, origin, voxel_size):
    """lrf_mesh_cells on one brick: values [dx, dy, dz] fp32 at lattice points lo + (x, y, z).
    -> (edges {edge key: vertex [3] f32}, triangles [(sort key, edge key, edge key, edge key)]).  Triangles are wound
    counter-clockwise seen from outside (the right-hand normal points to lower values)."""
    values = np.asarray(values, np.float32)
    d = values.shape
    ins = values >= np.float32(level)
    idx = np.zeros([n - 1 for n in d], np.int64)
    for c, (ox, oy, oz) in enumerate(CORNERS):
        idx |= ins[ox:ox + d[0] - 1, oy:oy + d[1] - 1, oz:oz + d[2] - 1].astype(np.int64) << c
    edges, tris = {}, []
    for x, y, z in zip(*np.nonzero((idx != 0) & (idx != 255))):
        row = TRI_TABLE[idx[x, y, z]]
        keys = {}
        for e in set(row):
            ca, cb = EDGES[e]
            pa = np.add((x, y, z), CORNERS[ca])
            pb = np.add((x, y, z), CORNERS[cb])
            lo_pt, hi_pt = (pa, pb) if tuple(pa) < tuple(pb) else (pb, pa)
            axis = int(np.argmax(hi_pt - lo_pt))
            gi = [int(lo_pt[a]) + int(lo[a]) for a in range(3)]
            k = edge_key(gi, axis)
            keys[e] = k
            if k not in edges:
                edges[k] = edge_vertex(gi, axis, values[tuple(lo_pt)], values[tuple(hi_pt)], level, origin, voxel_size)
        ck = cell_key((x + lo[0], y + lo[1], z + lo[2]))
        for t in range(len(row) // 3):
            e0, e1, e2 = row[3 * t:3 * t + 3]
            tris.append(((ck << 3) | t, keys[e0], keys[e2], keys[e1]))
    return edges, tris


def extract(edges, tris):
    """lrf_mesh_extract: vertices in ascending edge-key order, triangles in ascending sort-key order as vertex ranks.
    -> (xyz [V, 3] float32, faces [T, 3] int32)."""
    keys = sorted(edges)
    rank = {k: r for r, k in enumerate(keys)}
    xyz = np.array([edges[k] for k in keys], np.float32).reshape(-1, 3)
    faces = np.array([[rank[a], rank[b], rank[c]] for _, a, b, c in sorted(tris)], np.int32).reshape(-1, 3)
    return xyz, faces


def merge(parts):
    """cells() of several bricks -> one (edges, triangles): an edge shared by two bricks gets the same bits in both."""
    edges, tris = {}, []
    for e, t in parts:
        for k, v in e.items():
            assert k not in edges or edges[k].tobytes() == v.tobytes()
            edges[k] = v
        tris += t
    return edges, tris


def mesh_lattice(values, lo, level, origin, voxel_size):
    """cells + extract of one brick -> (xyz, faces)."""
    return extract(*cells(values, lo, level, origin, voxel_size))


# ---- the same restatement, vectorised ----------------------------------------------------------------------------
# TRI_TABLE as a [256, 16] array (-1 after the last edge), and per edge its lower corner's offset and its axis
TRI_NP = np.array([r + [-1] * (16 - len(r)) for r in TRI_TABLE], np.int8)
EDGE_OFF = np.array([np.minimum(CORNERS[a], CORNERS[b]) for a, b in EDGES], np.int32)
EDGE_AXIS = np.array([int(np.argmax(np.abs(np.subtract(CORNERS[b], CORNERS[a])))) for a, b in EDGES], np.int32)
WINDING = np.array([0, 2, 1], np.int32)                  # (e0, e2, e1): the outward winding
SLAB_CELLS = 1 << 20                                     # cells per x-slab of cells_parts


def _keys_np(g, shifts):
    """Keys of lattice indices g [..., 3] (each in [-2^19, 2^19)): (g_a + 2^19) << shifts[a], or-ed -> uint64."""
    out = np.zeros(g.shape[:-1], np.uint64)
    for a in range(3):
        out |= (g[..., a].astype(np.int64) + HALF).astype(np.uint64) << np.uint64(shifts[a])
    return out


def cells_parts(values, lo, level, origin, voxel_size):
    """cells() vectorised, one x-slab of cells at a time so its memory stays bounded.  -> (edge keys [E] uint64,
    vertices [E, 3] float32, triangle sort keys [T] uint64, triangle edge keys [T, 3] uint64); an edge may appear
    once per slab, every time with the same vertex bits."""
    v = np.asarray(values, np.float32)
    d = v.shape
    ny, nz = d[1] - 1, d[2] - 1
    lvl, vs = np.float32(level), np.float32(voxel_size)
    org = np.asarray(origin, np.float32)
    lo = np.asarray(lo, np.int32)
    step = max(1, SLAB_CELLS // max(1, ny * nz))
    ek, ev, tk, te = [], [], [], []
    for x0 in range(0, d[0] - 1, step):
        x1 = min(x0 + step, d[0] - 1)
        ins = v[x0:x1 + 1] >= lvl                                       # NaN is outside
        idx = np.zeros((x1 - x0, ny, nz), np.uint8)
        for c, (ox, oy, oz) in enumerate(CORNERS):
            idx |= ins[ox:ox + x1 - x0, oy:oy + ny, oz:oz + nz].astype(np.uint8) << np.uint8(c)
        cell = np.stack(np.nonzero((idx != 0) & (idx != 255)), 1).astype(np.int32)
        if len(cell) == 0:
            continue
        case = idx[cell[:, 0], cell[:, 1], cell[:, 2]]
        cell[:, 0] += x0
        del idx, ins
        tri = TRI_NP[case]
        ci, k = np.nonzero(tri[:, 0:15:3] >= 0)
        e = tri[ci[:, None], 3 * k[:, None] + WINDING].astype(np.int32)  # [T, 3] the edges, outward winding
        del tri
        pt = cell[ci][:, None, :] + EDGE_OFF[e]                           # [T, 3, 3] lower points in the brick
        axis = EDGE_AXIS[e]
        keys = _keys_np(pt + lo, (42, 22, 2)) | axis.astype(np.uint64)
        tk.append((_keys_np(cell[ci] + lo, (40, 20, 0)) << np.uint64(3)) | k.astype(np.uint64))
        te.append(keys)
        uk, first = np.unique(keys.reshape(-1), return_index=True)
        lp, ax = pt.reshape(-1, 3)[first], axis.reshape(-1)[first]
        del pt, axis, e
        r = np.arange(len(ax))
        hp = lp.copy()
        hp[r, ax] += 1
        va, vb = v[lp[:, 0], lp[:, 1], lp[:, 2]], v[hp[:, 0], hp[:, 1], hp[:, 2]]
        with np.errstate(all="ignore"):
            t = (lvl - va) / (vb - va)
        t = np.where(np.isfinite(t), np.clip(t, np.float32(0), np.float32(1)), np.float32(0)).astype(np.float32)
        gl = lp + lo
        xyz = (org[None] + gl.astype(np.float32) * vs).astype(np.float32)
        pa = xyz[r, ax]
        pb = (org[ax] + (gl[r, ax] + 1).astype(np.float32) * vs).astype(np.float32)
        xyz[r, ax] = pa + t * (pb - pa)
        ek.append(uk)
        ev.append(xyz)
    cat = lambda parts, shape, dt: np.concatenate(parts) if parts else np.zeros(shape, dt)
    return (cat(ek, (0,), np.uint64), cat(ev, (0, 3), np.float32), cat(tk, (0,), np.uint64),
            cat(te, (0, 3), np.uint64))


def extract_np(parts):
    """extract() of the concatenation of cells_parts() of one or more bricks (merge(), then extract(), vectorised):
    each edge key's first vertex, in ascending key order, and the triangles in ascending sort-key order as vertex
    ranks.  -> (xyz [V, 3] float32, faces [T, 3] int32)."""
    keys = np.concatenate([p[0] for p in parts])
    uk, first = np.unique(keys, return_index=True)
    del keys
    xyz = np.concatenate([p[1] for p in parts])[first]
    tk = np.concatenate([p[2] for p in parts])
    order = np.argsort(tk, kind="stable")
    del tk
    te = np.concatenate([p[3] for p in parts])
    faces = np.empty((len(order), 3), np.int32)
    for i in range(0, len(order), 1 << 22):
        faces[i:i + (1 << 22)] = np.searchsorted(uk, te[order[i:i + (1 << 22)]])
    return xyz, faces


def cells_np(values, lo, level, origin, voxel_size):
    """mesh_lattice vectorised: the same (xyz, faces), bit for bit."""
    return extract_np([cells_parts(values, lo, level, origin, voxel_size)])


# ---- the owner rule and the table's slots ------------------------------------------------------------------------
def owner32(xyz, w2rf):
    """The owner rule of lrf_mesh_* in float32: per field k, y = float32(p) + float32(w_k) per axis; a field with a NaN
    component of y is skipped, the smallest max |y_a| wins strictly (exact ties to the lowest k, +inf never wins).
    -> (owner [M] int32, -1 when no field has a finite norm; its norm [M] float32, +inf there)."""
    p = np.asarray(xyz, np.float32).reshape(-1, 3)
    w = np.asarray(w2rf, np.float32).reshape(-1, 3)
    owner = np.full(len(p), -1, np.int32)
    best = np.full(len(p), np.inf, np.float32)
    for k in range(len(w)):
        y = p + w[k]
        with np.errstate(invalid="ignore"):
            n = np.abs(y).max(1)
            win = ~np.isnan(y).any(1) & (n < best)
        owner[win] = k
        best[win] = n[win]
    return owner, best


def probe_slots(keys, capacity):
    """The occupied slots of the edge table (csrc/lrf_table.cuh: linear probing from mix64(key) & (capacity - 1),
    wrapping to 0) after the distinct `keys` are claimed, in any order."""
    import export_oracle as eo
    return eo.probe_table(keys, capacity)


# ---- checks of a mesh --------------------------------------------------------------------------------------------
def directed_edges(faces):
    """{(a, b): uses} over the triangles' directed edges."""
    out = {}
    for f in faces:
        for j in range(3):
            e = (int(f[j]), int(f[(j + 1) % 3]))
            out[e] = out.get(e, 0) + 1
    return out


def is_closed_oriented(faces):
    """Every directed edge is used once and its reverse once: a closed, consistently oriented 2-manifold's edges."""
    d = directed_edges(faces)
    return all(m == 1 and d.get((b, a)) == 1 for (a, b), m in d.items())


def euler_characteristic(xyz, faces):
    """V - E + F over the vertices the faces use."""
    used = np.unique(faces)
    n_edges = len({(min(a, b), max(a, b)) for a, b in directed_edges(faces)})
    return len(used) - n_edges + len(faces)


def signed_volume(xyz, faces):
    """sum over triangles of v0 . (v1 x v2) / 6 in float64: the enclosed volume, positive for outward winding."""
    v = xyz.astype(np.float64)[faces]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6)


def read_mesh_ply(data):
    """(xyz, normals or None, rgb, faces or None) of a binary little-endian PLY as write_ply writes it."""
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0", lines[:2]
    n_v, n_f, props, face_prop = 0, None, [], None
    for l in lines[2:-1]:
        w = l.split()
        if w[0] == "element":
            if w[1] == "vertex":
                n_v = int(w[2])
            else:
                assert w[1] == "face"
                n_f = int(w[2])
        elif n_f is None:
            props.append((w[1], w[2]))
        else:
            face_prop = w[1:]
    names = [p[1] for p in props]
    assert all(t == "float" for t, _ in props[:-3]) and [t for t, _ in props[-3:]] == ["uchar"] * 3
    dt = [(nm, "<f4") for nm in names[:-3]] + [(nm, "u1") for nm in names[-3:]]
    v = np.frombuffer(data[end:end + n_v * np.dtype(dt).itemsize], dtype=dt)
    xyz = np.stack([v[c] for c in ("x", "y", "z")], 1)
    normals = np.stack([v[c] for c in ("nx", "ny", "nz")], 1) if "nx" in names else None
    rgb = np.stack([v[c] for c in ("red", "green", "blue")], 1)
    faces = None
    if n_f is not None:
        assert face_prop == ["list", "uchar", "int", "vertex_indices"]
        f = np.frombuffer(data[end + n_v * np.dtype(dt).itemsize:], dtype=[("n", "u1"), ("v", "<i4", (3,))])
        assert len(f) == n_f and (f["n"] == 3).all()
        faces = f["v"].copy()
    return xyz, normals, rgb, faces


# ---- the scalar field A in float64 -------------------------------------------------------------------------------
def mesh_value64(fields, steps, w2rf, p, max_norm):
    """A at world points p [M, 3] (float64 torch) from Field64 fields (render64.Field64), their stepSizes and world2rf
    [K, 3], every operation in float64 -> (A [M], owner [M] (-1: beyond max_norm), flagged [M]).  A point is flagged
    when its owner or its inside-the-cube decision lies within the fp32 error bound (two norms, or the norm and
    max_norm, closer than 2^-20 (1 + |p|), unless the two norms are the same coordinate of p plus the same world2rf
    component: that tie is exact in fp32 too and goes to the lower field), or when an alpha mask's value at it is within 1e-6 of 0 (the cull)."""
    import render64 as r64
    p = p.to(torch.float64)
    w = torch.as_tensor(np.asarray(w2rf, np.float64), device=p.device).reshape(-1, 3)
    x = p[:, None, :] + w[None]                                # [M, K, 3]
    norms = x.abs().amax(-1)
    srt = norms.sort(dim=-1, stable=True)                         # ties: the lower field first
    best, owner = srt.values[:, 0], srt.indices[:, 0]
    tol = 2.0 ** -20 * (1 + p.abs().amax(-1) + w.abs().max())
    flagged = (best - max_norm).abs() <= tol
    if norms.shape[1] > 1:
        # an exact tie taken from the same axis of two fields with the same world2rf there is exact in fp32 too
        k2 = srt.indices[:, 1]
        ax = x.abs().argmax(-1)
        a1, a2 = ax.gather(1, owner[:, None])[:, 0], ax.gather(1, k2[:, None])[:, 0]
        same = (a1 == a2) & (w[owner].gather(1, a1[:, None]) == w[k2].gather(1, a1[:, None]))[:, 0]
        diff = srt.values[:, 1] - best
        flagged |= (diff <= tol) & ~((diff == 0) & same)
    inside = best <= max_norm
    A = torch.zeros(p.shape[0], dtype=torch.float64, device=p.device)
    for k, F in enumerate(fields):
        sel = (owner == k) & inside
        if not sel.any():
            continue
        xk = x[sel, k]
        n = xk.abs().amax(-1, keepdim=True).clamp(min=1e-6)
        c = torch.where(n <= 1, xk, (2 * n - 1) / (n * n) * xk)
        q = (c - F.aabb[0]) * (2.0 / (F.aabb[1] - F.aabb[0])) - 1
        f = sum(r64._lookup(F.p[f"density_plane.{i}"].detach(), F.p[f"density_line.{i}"].detach(), q, i).sum(1)
                for i in range(3))
        sigma = Fn.softplus(f + F.shift) if F.act == "softplus" else Fn.relu(f)
        if F.alpha_vol is not None:
            mv, _ = r64._mask_value(F, c)
            sigma = torch.where(mv > 0, sigma, torch.zeros_like(sigma))
            fl = torch.zeros_like(flagged)
            fl[sel] = mv.abs() <= 1e-6
            flagged |= fl
        A[sel] = 1 - torch.exp(-sigma * float(steps[k]))
    owner = torch.where(inside, owner, torch.full_like(owner, -1))
    return A, owner, flagged
