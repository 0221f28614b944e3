// lrf_mesh.cu -- the scene's surface as a triangle mesh: marching cubes over the fields' density on a world-space
// lattice, on the device.
//
// lrf_mesh_lattice writes A (mesh_value below: the nearest-centre field's getDenseAlpha value) at every point of one
// brick of the lattice.  lrf_mesh_cells runs the 256-case table over the brick's cells: each cut edge is claimed once
// in an open-addressing table keyed by its lower lattice point and axis, and stores its vertex; each triangle is
// appended with the slots of its edges.  lrf_mesh_extract sorts the edges by key and the triangles by (cell, index in
// the case) with a radix sort, so the mesh comes out in one canonical order whatever the brick size, the brick
// order or the thread scheduling.  lrf_mesh_normals takes the normals from central differences of A.  The edge
// table's conventions are lrf_table.cuh's; the sort is KeySlotSort.
//
// The lattice points and vertices are written with explicit round-to-nearest fp32 operations (no FMA contraction), so
// a numpy float32 restatement reproduces them bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/localrf_b200.h"
#include "lrf_device.cuh"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"
#include "lrf_table.cuh"

namespace lrf {

namespace {

constexpr int MC_THREADS = 256;
constexpr int KEY_HALF = 1 << 19;       // lattice indices lie in [-2^19, 2^19): 20 bits per axis

// The widely published 256-case triangle table (three edges per triangle, -1 after the last).  Bit c of the case is
// set when corner c is inside; corners 0-3 are (0,0,0), (1,0,0), (1,1,0), (0,1,0) and 4-7 the same at z = 1.  The
// table resolves an ambiguous face from the face's corners alone, so the two cells that share it agree.
__constant__ signed char TRI[256][16] = {
    {-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {0,1,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,8,3,9,8,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,2,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,1,2,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {9,2,10,0,2,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {2,8,3,2,10,8,10,9,8,-1,-1,-1,-1,-1,-1,-1},
    {3,11,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,11,2,8,11,0,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,9,0,2,3,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,11,2,1,9,11,9,8,11,-1,-1,-1,-1,-1,-1,-1},
    {3,10,1,11,10,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,10,1,0,8,10,8,11,10,-1,-1,-1,-1,-1,-1,-1},
    {3,9,0,3,11,9,11,10,9,-1,-1,-1,-1,-1,-1,-1}, {9,8,10,10,8,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,7,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,3,0,7,3,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {0,1,9,8,4,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,1,9,4,7,1,7,3,1,-1,-1,-1,-1,-1,-1,-1},
    {1,2,10,8,4,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,4,7,3,0,4,1,2,10,-1,-1,-1,-1,-1,-1,-1},
    {9,2,10,9,0,2,8,4,7,-1,-1,-1,-1,-1,-1,-1}, {2,10,9,2,9,7,2,7,3,7,9,4,-1,-1,-1,-1},
    {8,4,7,3,11,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {11,4,7,11,2,4,2,0,4,-1,-1,-1,-1,-1,-1,-1},
    {9,0,1,8,4,7,2,3,11,-1,-1,-1,-1,-1,-1,-1}, {4,7,11,9,4,11,9,11,2,9,2,1,-1,-1,-1,-1},
    {3,10,1,3,11,10,7,8,4,-1,-1,-1,-1,-1,-1,-1}, {1,11,10,1,4,11,1,0,4,7,11,4,-1,-1,-1,-1},
    {4,7,8,9,0,11,9,11,10,11,0,3,-1,-1,-1,-1}, {4,7,11,4,11,9,9,11,10,-1,-1,-1,-1,-1,-1,-1},
    {9,5,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {9,5,4,0,8,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {0,5,4,1,5,0,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {8,5,4,8,3,5,3,1,5,-1,-1,-1,-1,-1,-1,-1},
    {1,2,10,9,5,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,0,8,1,2,10,4,9,5,-1,-1,-1,-1,-1,-1,-1},
    {5,2,10,5,4,2,4,0,2,-1,-1,-1,-1,-1,-1,-1}, {2,10,5,3,2,5,3,5,4,3,4,8,-1,-1,-1,-1},
    {9,5,4,2,3,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,11,2,0,8,11,4,9,5,-1,-1,-1,-1,-1,-1,-1},
    {0,5,4,0,1,5,2,3,11,-1,-1,-1,-1,-1,-1,-1}, {2,1,5,2,5,8,2,8,11,4,8,5,-1,-1,-1,-1},
    {10,3,11,10,1,3,9,5,4,-1,-1,-1,-1,-1,-1,-1}, {4,9,5,0,8,1,8,10,1,8,11,10,-1,-1,-1,-1},
    {5,4,0,5,0,11,5,11,10,11,0,3,-1,-1,-1,-1}, {5,4,8,5,8,10,10,8,11,-1,-1,-1,-1,-1,-1,-1},
    {9,7,8,5,7,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {9,3,0,9,5,3,5,7,3,-1,-1,-1,-1,-1,-1,-1},
    {0,7,8,0,1,7,1,5,7,-1,-1,-1,-1,-1,-1,-1}, {1,5,3,3,5,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {9,7,8,9,5,7,10,1,2,-1,-1,-1,-1,-1,-1,-1}, {10,1,2,9,5,0,5,3,0,5,7,3,-1,-1,-1,-1},
    {8,0,2,8,2,5,8,5,7,10,5,2,-1,-1,-1,-1}, {2,10,5,2,5,3,3,5,7,-1,-1,-1,-1,-1,-1,-1},
    {7,9,5,7,8,9,3,11,2,-1,-1,-1,-1,-1,-1,-1}, {9,5,7,9,7,2,9,2,0,2,7,11,-1,-1,-1,-1},
    {2,3,11,0,1,8,1,7,8,1,5,7,-1,-1,-1,-1}, {11,2,1,11,1,7,7,1,5,-1,-1,-1,-1,-1,-1,-1},
    {9,5,8,8,5,7,10,1,3,10,3,11,-1,-1,-1,-1}, {5,7,0,5,0,9,7,11,0,1,0,10,11,10,0,-1},
    {11,10,0,11,0,3,10,5,0,8,0,7,5,7,0,-1}, {11,10,5,7,11,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {10,6,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,5,10,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {9,0,1,5,10,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,8,3,1,9,8,5,10,6,-1,-1,-1,-1,-1,-1,-1},
    {1,6,5,2,6,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,6,5,1,2,6,3,0,8,-1,-1,-1,-1,-1,-1,-1},
    {9,6,5,9,0,6,0,2,6,-1,-1,-1,-1,-1,-1,-1}, {5,9,8,5,8,2,5,2,6,3,2,8,-1,-1,-1,-1},
    {2,3,11,10,6,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {11,0,8,11,2,0,10,6,5,-1,-1,-1,-1,-1,-1,-1},
    {0,1,9,2,3,11,5,10,6,-1,-1,-1,-1,-1,-1,-1}, {5,10,6,1,9,2,9,11,2,9,8,11,-1,-1,-1,-1},
    {6,3,11,6,5,3,5,1,3,-1,-1,-1,-1,-1,-1,-1}, {0,8,11,0,11,5,0,5,1,5,11,6,-1,-1,-1,-1},
    {3,11,6,0,3,6,0,6,5,0,5,9,-1,-1,-1,-1}, {6,5,9,6,9,11,11,9,8,-1,-1,-1,-1,-1,-1,-1},
    {5,10,6,4,7,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,3,0,4,7,3,6,5,10,-1,-1,-1,-1,-1,-1,-1},
    {1,9,0,5,10,6,8,4,7,-1,-1,-1,-1,-1,-1,-1}, {10,6,5,1,9,7,1,7,3,7,9,4,-1,-1,-1,-1},
    {6,1,2,6,5,1,4,7,8,-1,-1,-1,-1,-1,-1,-1}, {1,2,5,5,2,6,3,0,4,3,4,7,-1,-1,-1,-1},
    {8,4,7,9,0,5,0,6,5,0,2,6,-1,-1,-1,-1}, {7,3,9,7,9,4,3,2,9,5,9,6,2,6,9,-1},
    {3,11,2,7,8,4,10,6,5,-1,-1,-1,-1,-1,-1,-1}, {5,10,6,4,7,2,4,2,0,2,7,11,-1,-1,-1,-1},
    {0,1,9,4,7,8,2,3,11,5,10,6,-1,-1,-1,-1}, {9,2,1,9,11,2,9,4,11,7,11,4,5,10,6,-1},
    {8,4,7,3,11,5,3,5,1,5,11,6,-1,-1,-1,-1}, {5,1,11,5,11,6,1,0,11,7,11,4,0,4,11,-1},
    {0,5,9,0,6,5,0,3,6,11,6,3,8,4,7,-1}, {6,5,9,6,9,11,4,7,9,7,11,9,-1,-1,-1,-1},
    {10,4,9,6,4,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,10,6,4,9,10,0,8,3,-1,-1,-1,-1,-1,-1,-1},
    {10,0,1,10,6,0,6,4,0,-1,-1,-1,-1,-1,-1,-1}, {8,3,1,8,1,6,8,6,4,6,1,10,-1,-1,-1,-1},
    {1,4,9,1,2,4,2,6,4,-1,-1,-1,-1,-1,-1,-1}, {3,0,8,1,2,9,2,4,9,2,6,4,-1,-1,-1,-1},
    {0,2,4,4,2,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {8,3,2,8,2,4,4,2,6,-1,-1,-1,-1,-1,-1,-1},
    {10,4,9,10,6,4,11,2,3,-1,-1,-1,-1,-1,-1,-1}, {0,8,2,2,8,11,4,9,10,4,10,6,-1,-1,-1,-1},
    {3,11,2,0,1,6,0,6,4,6,1,10,-1,-1,-1,-1}, {6,4,1,6,1,10,4,8,1,2,1,11,8,11,1,-1},
    {9,6,4,9,3,6,9,1,3,11,6,3,-1,-1,-1,-1}, {8,11,1,8,1,0,11,6,1,9,1,4,6,4,1,-1},
    {3,11,6,3,6,0,0,6,4,-1,-1,-1,-1,-1,-1,-1}, {6,4,8,11,6,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {7,10,6,7,8,10,8,9,10,-1,-1,-1,-1,-1,-1,-1}, {0,7,3,0,10,7,0,9,10,6,7,10,-1,-1,-1,-1},
    {10,6,7,1,10,7,1,7,8,1,8,0,-1,-1,-1,-1}, {10,6,7,10,7,1,1,7,3,-1,-1,-1,-1,-1,-1,-1},
    {1,2,6,1,6,8,1,8,9,8,6,7,-1,-1,-1,-1}, {2,6,9,2,9,1,6,7,9,0,9,3,7,3,9,-1},
    {7,8,0,7,0,6,6,0,2,-1,-1,-1,-1,-1,-1,-1}, {7,3,2,6,7,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {2,3,11,10,6,8,10,8,9,8,6,7,-1,-1,-1,-1}, {2,0,7,2,7,11,0,9,7,6,7,10,9,10,7,-1},
    {1,8,0,1,7,8,1,10,7,6,7,10,2,3,11,-1}, {11,2,1,11,1,7,10,6,1,6,7,1,-1,-1,-1,-1},
    {8,9,6,8,6,7,9,1,6,11,6,3,1,3,6,-1}, {0,9,1,11,6,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {7,8,0,7,0,6,3,11,0,11,6,0,-1,-1,-1,-1}, {7,11,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {7,6,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,0,8,11,7,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {0,1,9,11,7,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {8,1,9,8,3,1,11,7,6,-1,-1,-1,-1,-1,-1,-1},
    {10,1,2,6,11,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,2,10,3,0,8,6,11,7,-1,-1,-1,-1,-1,-1,-1},
    {2,9,0,2,10,9,6,11,7,-1,-1,-1,-1,-1,-1,-1}, {6,11,7,2,10,3,10,8,3,10,9,8,-1,-1,-1,-1},
    {7,2,3,6,2,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {7,0,8,7,6,0,6,2,0,-1,-1,-1,-1,-1,-1,-1},
    {2,7,6,2,3,7,0,1,9,-1,-1,-1,-1,-1,-1,-1}, {1,6,2,1,8,6,1,9,8,8,7,6,-1,-1,-1,-1},
    {10,7,6,10,1,7,1,3,7,-1,-1,-1,-1,-1,-1,-1}, {10,7,6,1,7,10,1,8,7,1,0,8,-1,-1,-1,-1},
    {0,3,7,0,7,10,0,10,9,6,10,7,-1,-1,-1,-1}, {7,6,10,7,10,8,8,10,9,-1,-1,-1,-1,-1,-1,-1},
    {6,8,4,11,8,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,6,11,3,0,6,0,4,6,-1,-1,-1,-1,-1,-1,-1},
    {8,6,11,8,4,6,9,0,1,-1,-1,-1,-1,-1,-1,-1}, {9,4,6,9,6,3,9,3,1,11,3,6,-1,-1,-1,-1},
    {6,8,4,6,11,8,2,10,1,-1,-1,-1,-1,-1,-1,-1}, {1,2,10,3,0,11,0,6,11,0,4,6,-1,-1,-1,-1},
    {4,11,8,4,6,11,0,2,9,2,10,9,-1,-1,-1,-1}, {10,9,3,10,3,2,9,4,3,11,3,6,4,6,3,-1},
    {8,2,3,8,4,2,4,6,2,-1,-1,-1,-1,-1,-1,-1}, {0,4,2,4,6,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,9,0,2,3,4,2,4,6,4,3,8,-1,-1,-1,-1}, {1,9,4,1,4,2,2,4,6,-1,-1,-1,-1,-1,-1,-1},
    {8,1,3,8,6,1,8,4,6,6,10,1,-1,-1,-1,-1}, {10,1,0,10,0,6,6,0,4,-1,-1,-1,-1,-1,-1,-1},
    {4,6,3,4,3,8,6,10,3,0,3,9,10,9,3,-1}, {10,9,4,6,10,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,9,5,7,6,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,4,9,5,11,7,6,-1,-1,-1,-1,-1,-1,-1},
    {5,0,1,5,4,0,7,6,11,-1,-1,-1,-1,-1,-1,-1}, {11,7,6,8,3,4,3,5,4,3,1,5,-1,-1,-1,-1},
    {9,5,4,10,1,2,7,6,11,-1,-1,-1,-1,-1,-1,-1}, {6,11,7,1,2,10,0,8,3,4,9,5,-1,-1,-1,-1},
    {7,6,11,5,4,10,4,2,10,4,0,2,-1,-1,-1,-1}, {3,4,8,3,5,4,3,2,5,10,5,2,11,7,6,-1},
    {7,2,3,7,6,2,5,4,9,-1,-1,-1,-1,-1,-1,-1}, {9,5,4,0,8,6,0,6,2,6,8,7,-1,-1,-1,-1},
    {3,6,2,3,7,6,1,5,0,5,4,0,-1,-1,-1,-1}, {6,2,8,6,8,7,2,1,8,4,8,5,1,5,8,-1},
    {9,5,4,10,1,6,1,7,6,1,3,7,-1,-1,-1,-1}, {1,6,10,1,7,6,1,0,7,8,7,0,9,5,4,-1},
    {4,0,10,4,10,5,0,3,10,6,10,7,3,7,10,-1}, {7,6,10,7,10,8,5,4,10,4,8,10,-1,-1,-1,-1},
    {6,9,5,6,11,9,11,8,9,-1,-1,-1,-1,-1,-1,-1}, {3,6,11,0,6,3,0,5,6,0,9,5,-1,-1,-1,-1},
    {0,11,8,0,5,11,0,1,5,5,6,11,-1,-1,-1,-1}, {6,11,3,6,3,5,5,3,1,-1,-1,-1,-1,-1,-1,-1},
    {1,2,10,9,5,11,9,11,8,11,5,6,-1,-1,-1,-1}, {0,11,3,0,6,11,0,9,6,5,6,9,1,2,10,-1},
    {11,8,5,11,5,6,8,0,5,10,5,2,0,2,5,-1}, {6,11,3,6,3,5,2,10,3,10,5,3,-1,-1,-1,-1},
    {5,8,9,5,2,8,5,6,2,3,8,2,-1,-1,-1,-1}, {9,5,6,9,6,0,0,6,2,-1,-1,-1,-1,-1,-1,-1},
    {1,5,8,1,8,0,5,6,8,3,8,2,6,2,8,-1}, {1,5,6,2,1,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,3,6,1,6,10,3,8,6,5,6,9,8,9,6,-1}, {10,1,0,10,0,6,9,5,0,5,6,0,-1,-1,-1,-1},
    {0,3,8,5,6,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {10,5,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {11,5,10,7,5,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {11,5,10,11,7,5,8,3,0,-1,-1,-1,-1,-1,-1,-1},
    {5,11,7,5,10,11,1,9,0,-1,-1,-1,-1,-1,-1,-1}, {10,7,5,10,11,7,9,8,1,8,3,1,-1,-1,-1,-1},
    {11,1,2,11,7,1,7,5,1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,1,2,7,1,7,5,7,2,11,-1,-1,-1,-1},
    {9,7,5,9,2,7,9,0,2,2,11,7,-1,-1,-1,-1}, {7,5,2,7,2,11,5,9,2,3,2,8,9,8,2,-1},
    {2,5,10,2,3,5,3,7,5,-1,-1,-1,-1,-1,-1,-1}, {8,2,0,8,5,2,8,7,5,10,2,5,-1,-1,-1,-1},
    {9,0,1,5,10,3,5,3,7,3,10,2,-1,-1,-1,-1}, {9,8,2,9,2,1,8,7,2,10,2,5,7,5,2,-1},
    {1,3,5,3,7,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,7,0,7,1,1,7,5,-1,-1,-1,-1,-1,-1,-1},
    {9,0,3,9,3,5,5,3,7,-1,-1,-1,-1,-1,-1,-1}, {9,8,7,5,9,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {5,8,4,5,10,8,10,11,8,-1,-1,-1,-1,-1,-1,-1}, {5,0,4,5,11,0,5,10,11,11,3,0,-1,-1,-1,-1},
    {0,1,9,8,4,10,8,10,11,10,4,5,-1,-1,-1,-1}, {10,11,4,10,4,5,11,3,4,9,4,1,3,1,4,-1},
    {2,5,1,2,8,5,2,11,8,4,5,8,-1,-1,-1,-1}, {0,4,11,0,11,3,4,5,11,2,11,1,5,1,11,-1},
    {0,2,5,0,5,9,2,11,5,4,5,8,11,8,5,-1}, {9,4,5,2,11,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {2,5,10,3,5,2,3,4,5,3,8,4,-1,-1,-1,-1}, {5,10,2,5,2,4,4,2,0,-1,-1,-1,-1,-1,-1,-1},
    {3,10,2,3,5,10,3,8,5,4,5,8,0,1,9,-1}, {5,10,2,5,2,4,1,9,2,9,4,2,-1,-1,-1,-1},
    {8,4,5,8,5,3,3,5,1,-1,-1,-1,-1,-1,-1,-1}, {0,4,5,1,0,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {8,4,5,8,5,3,9,0,5,0,3,5,-1,-1,-1,-1}, {9,4,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,11,7,4,9,11,9,10,11,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,4,9,7,9,11,7,9,10,11,-1,-1,-1,-1},
    {1,10,11,1,11,4,1,4,0,7,4,11,-1,-1,-1,-1}, {3,1,4,3,4,8,1,10,4,7,4,11,10,11,4,-1},
    {4,11,7,9,11,4,9,2,11,9,1,2,-1,-1,-1,-1}, {9,7,4,9,11,7,9,1,11,2,11,1,0,8,3,-1},
    {11,7,4,11,4,2,2,4,0,-1,-1,-1,-1,-1,-1,-1}, {11,7,4,11,4,2,8,3,4,3,2,4,-1,-1,-1,-1},
    {2,9,10,2,7,9,2,3,7,7,4,9,-1,-1,-1,-1}, {9,10,7,9,7,4,10,2,7,8,7,0,2,0,7,-1},
    {3,7,10,3,10,2,7,4,10,1,10,0,4,0,10,-1}, {1,10,2,8,7,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {4,9,1,4,1,7,7,1,3,-1,-1,-1,-1,-1,-1,-1}, {4,9,1,4,1,7,0,8,1,8,7,1,-1,-1,-1,-1},
    {4,0,3,7,4,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,8,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {9,10,8,10,11,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,0,9,3,9,11,11,9,10,-1,-1,-1,-1,-1,-1,-1},
    {0,1,10,0,10,8,8,10,11,-1,-1,-1,-1,-1,-1,-1}, {3,1,10,11,3,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,2,11,1,11,9,9,11,8,-1,-1,-1,-1,-1,-1,-1}, {3,0,9,3,9,11,1,2,9,2,11,9,-1,-1,-1,-1},
    {0,2,11,8,0,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,2,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {2,3,8,2,8,10,10,8,9,-1,-1,-1,-1,-1,-1,-1}, {9,10,2,0,9,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {2,3,8,2,8,10,0,1,8,1,10,8,-1,-1,-1,-1}, {1,10,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {1,3,8,9,1,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1},
    {0,3,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}
};

// Edge e joins corner edge_lo(e) to corner edge_hi(e) along axis edge_axis(e), the lower point first; nibble e of
// each constant, for edges 0-11: lo 0 1 3 0 4 5 7 4 0 1 2 3, hi 1 2 2 3 5 6 6 7 4 5 6 7, axis 0 1 0 1 0 1 0 1 2 2 2 2.
__host__ __device__ constexpr int edge_lo(int e) { return (int)((0x321047540310ull >> (4 * e)) & 15); }
__host__ __device__ constexpr int edge_hi(int e) { return (int)((0x765476653221ull >> (4 * e)) & 15); }
__host__ __device__ constexpr int edge_axis(int e) { return (int)((0x222210101010ull >> (4 * e)) & 15); }
__host__ __device__ constexpr int corner_x(int c) { return (c ^ (c >> 1)) & 1; }
__host__ __device__ constexpr int corner_y(int c) { return (c >> 1) & 1; }
__host__ __device__ constexpr int corner_z(int c) { return (c >> 2) & 1; }

// origin_a + i voxel_size
__device__ __forceinline__ float lattice_coord(const MeshSceneDev& S, int a, int i) {
  return __fadd_rn(S.origin[a], __fmul_rn((float)i, S.voxel));
}

// The owner of world point p: the field with the smallest max-norm of x = p + world2rf_k (ties to the lowest k, a
// field with a NaN coordinate never wins) -> its index (-1 when no norm is below +inf), x in its frame and the norm.
__device__ __forceinline__ int mesh_owner(const MeshSceneDev& S, const float* p, float* x, float& norm) {
  int best = -1;
  norm = INFINITY;
  for (int k = 0; k < S.n_fields; ++k) {
    float y[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) y[a] = __fadd_rn(p[a], __ldg(S.w2rf + 3 * k + a));
    if (isnan(y[0]) || isnan(y[1]) || isnan(y[2])) continue;
    const float n = fmaxf(fmaxf(fabsf(y[0]), fabsf(y[1])), fabsf(y[2]));
    if (n < norm) {
      norm = n;
      best = k;
      x[0] = y[0]; x[1] = y[1]; x[2] = y[2];
    }
  }
  return best;
}

// A(p): the owner's getDenseAlpha value at contract(p + world2rf_owner); 0 beyond max_norm
__device__ __forceinline__ float mesh_value(const MeshSceneDev& S, const float* p) {
  float x[3], norm;
  const int k = mesh_owner(S, p, x, norm);
  if (k < 0 || !(norm <= S.max_norm)) return 0.0f;
  contract(x[0], x[1], x[2]);
  return dense_alpha_at(S.f[k], x, S.length[k]);
}

__global__ void __launch_bounds__(MC_THREADS) mesh_lattice_kernel(const __grid_constant__ MeshSceneDev S, int3 lo,
                                                                  int3 d, float* __restrict__ values) {
  const long long e = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
  if (e >= (long long)d.x * d.y * d.z) return;
  const int z = (int)(e % d.z), y = (int)((e / d.z) % d.y), x = (int)(e / ((long long)d.z * d.y));
  const float p[3] = {lattice_coord(S, 0, lo.x + x), lattice_coord(S, 1, lo.y + y), lattice_coord(S, 2, lo.z + z)};
  values[e] = mesh_value(S, p);
}

// slot[e] by selects, so the array stays in registers
__device__ __forceinline__ int pick(const int (&slot)[12], int e) {
  int r = -1;
#pragma unroll
  for (int ed = 0; ed < 12; ++ed) r = e == ed ? slot[ed] : r;
  return r;
}

// One thread per cell of the brick: its case, the vertices of its cut edges, its triangles.  The edge table's claim
// counter is stats[0]; the thread that claims an edge's slot stores its vertex there.
__global__ void __launch_bounds__(MC_THREADS) mesh_cells_kernel(const __grid_constant__ MeshSceneDev S, int3 lo,
                                                                int3 d, const float* __restrict__ values,
                                                                const LrfMeshTable t) {
  const int nx = d.x - 1, ny = d.y - 1, nz = d.z - 1;
  const long long e = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
  if (e >= (long long)nx * ny * nz || table_full(t.stats, t.capacity)) return;
  const int cz = (int)(e % nz), cy = (int)((e / nz) % ny), cx = (int)(e / ((long long)nz * ny));
  float v[8];
  int cube = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    v[c] = __ldg(values + ((long long)(cx + corner_x(c)) * d.y + cy + corner_y(c)) * d.z + cz + corner_z(c));
    cube |= (v[c] >= S.level ? 1 : 0) << c;                    // NaN is outside
  }
  if (cube == 0 || cube == 255) return;
  const int g[3] = {lo.x + cx, lo.y + cy, lo.z + cz};         // the cell's lower lattice point
  int slot[12];
#pragma unroll
  for (int ed = 0; ed < 12; ++ed) {
    const int a = edge_lo(ed), b = edge_hi(ed), axis = edge_axis(ed);
    slot[ed] = -1;
    if (((cube >> a) ^ (cube >> b)) & 1) {
      const int i[3] = {g[0] + corner_x(a), g[1] + corner_y(a), g[2] + corner_z(a)};
      float p[3] = {lattice_coord(S, 0, i[0]), lattice_coord(S, 1, i[1]), lattice_coord(S, 2, i[2])};
      const float pb = lattice_coord(S, axis, i[axis] + 1);
      float tt = __fdiv_rn(__fsub_rn(S.level, v[a]), __fsub_rn(v[b], v[a]));
      tt = isfinite(tt) ? fminf(fmaxf(tt, 0.0f), 1.0f) : 0.0f;
      p[axis] = __fadd_rn(p[axis], __fmul_rn(tt, __fsub_rn(pb, p[axis])));
      const unsigned long long key = ((unsigned long long)(i[0] + KEY_HALF) << 42) |
                                     ((unsigned long long)(i[1] + KEY_HALF) << 22) |
                                     ((unsigned long long)(i[2] + KEY_HALF) << 2) | (unsigned long long)axis;
      slot[ed] = find_or_claim(t.keys, t.capacity, t.stats, key, [&](unsigned long long s, bool claimed) {
        if (claimed) { t.verts[3 * s] = p[0]; t.verts[3 * s + 1] = p[1]; t.verts[3 * s + 2] = p[2]; }
      });
    }
  }
  const unsigned long long ck = ((unsigned long long)(g[0] + KEY_HALF) << 40) |
                                ((unsigned long long)(g[1] + KEY_HALF) << 20) | (unsigned long long)(g[2] + KEY_HALF);
  for (int k = 0; k < 5 && TRI[cube][3 * k] >= 0; ++k) {
    // the table's triangles face the inside; (e0, e2, e1) faces the outside
    const int s0 = pick(slot, TRI[cube][3 * k]), s1 = pick(slot, TRI[cube][3 * k + 2]),
              s2 = pick(slot, TRI[cube][3 * k + 1]);
    if (s0 < 0 || s1 < 0 || s2 < 0) return;
    const unsigned long long n = atomicAdd(t.stats + 1, 1ull);
    if (n >= (unsigned long long)t.max_triangles) return;    // more than max_triangles: overflow
    t.tri_keys[n] = (ck << 3) | (unsigned long long)k;
    t.tri_slots[3 * n] = s0; t.tri_slots[3 * n + 1] = s1; t.tri_slots[3 * n + 2] = s2;
  }
}

// sort inputs: the edge key of every claimed slot (NO_KEY, sorted last, for the others) ...
__global__ void __launch_bounds__(MC_THREADS) edge_keys_kernel(const LrfMeshTable t, unsigned long long* keys,
                                                               unsigned int* slots) {
  const long long i = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
  if (i >= t.capacity) return;
  const unsigned long long tag = t.keys[i];
  keys[i] = tag != 0 ? tag - 1 : NO_KEY;
  slots[i] = (unsigned int)i;
}

// ... and the sort key of every appended triangle
__global__ void __launch_bounds__(MC_THREADS) tri_keys_kernel(const LrfMeshTable t, unsigned long long* keys,
                                                              unsigned int* ids) {
  const long long i = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
  if (i >= t.max_triangles) return;
  keys[i] = (unsigned long long)i < t.stats[1] ? t.tri_keys[i] : NO_KEY;
  ids[i] = (unsigned int)i;
}

// vertex i of the sorted edges -> xyz row i, and its rank into the slot's entry of `rank`
__global__ void __launch_bounds__(MC_THREADS) vertex_write_kernel(const LrfMeshTable t, const unsigned long long* keys,
                                                                  const unsigned int* slots, float* xyz, int* rank,
                                                                  long long* counts) {
  const long long i = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
  if (i == 0) counts[0] = (long long)t.stats[0];
  if (i >= (t.capacity >> 1) || keys[i] == NO_KEY) return;
  const unsigned int s = slots[i];
  xyz[3 * i] = t.verts[3ull * s]; xyz[3 * i + 1] = t.verts[3ull * s + 1]; xyz[3 * i + 2] = t.verts[3ull * s + 2];
  rank[s] = (int)i;
}

// triangle i of the sorted triangles -> faces row i as vertex ranks
__global__ void __launch_bounds__(MC_THREADS) face_write_kernel(const LrfMeshTable t, const unsigned long long* keys,
                                                                const unsigned int* ids, const int* rank, int* faces,
                                                                long long* counts) {
  const long long i = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
  if (i == 0) counts[1] = (long long)t.stats[1];
  if (i >= t.max_triangles || keys[i] == NO_KEY) return;
  const long long j = ids[i];
#pragma unroll
  for (int c = 0; c < 3; ++c) faces[3 * i + c] = rank[t.tri_slots[3 * j + c]];
}

// per vertex: the outward normal from central differences of A, and the owner field
__global__ void __launch_bounds__(MC_THREADS) mesh_normals_kernel(const __grid_constant__ MeshSceneDev S,
                                                                  const float* __restrict__ xyz, long long n,
                                                                  float* __restrict__ normals, int* __restrict__ owner) {
  const long long i = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
  if (i >= n) return;
  const float x[3] = {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
  const float h = __fmul_rn(S.voxel, 0.5f);
  float g[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float p[3] = {x[0], x[1], x[2]};
    p[a] = __fadd_rn(x[a], h);
    const float hi = mesh_value(S, p);
    p[a] = __fsub_rn(x[a], h);
    g[a] = __fsub_rn(hi, mesh_value(S, p));
  }
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2])));
  const bool ok = len > 0.0f && isfinite(len);
#pragma unroll
  for (int a = 0; a < 3; ++a) normals[3 * i + a] = ok ? -__fdiv_rn(g[a], len) : 0.0f;
  float y[3], norm;
  owner[i] = mesh_owner(S, x, y, norm);
}

}  // namespace

cudaError_t launch_mesh_lattice(const MeshSceneDev& S, const int* lo, const int* dims, float* values,
                                cudaStream_t stream) {
  mesh_lattice_kernel<<<item_ctas((long long)dims[0] * dims[1] * dims[2], MC_THREADS), MC_THREADS, 0, stream>>>(
      S, make_int3(lo[0], lo[1], lo[2]), make_int3(dims[0], dims[1], dims[2]), values);
  return cudaGetLastError();
}

cudaError_t launch_mesh_cells(const MeshSceneDev& S, const int* lo, const int* dims, const float* values,
                              const LrfMeshTable& t, cudaStream_t stream) {
  const long long cells = (long long)(dims[0] - 1) * (dims[1] - 1) * (dims[2] - 1);
  mesh_cells_kernel<<<item_ctas(cells, MC_THREADS), MC_THREADS, 0, stream>>>(
      S, make_int3(lo[0], lo[1], lo[2]), make_int3(dims[0], dims[1], dims[2]), values, t);
  return cudaGetLastError();
}

// the sort's buffers of the edge keys and slots, the vertex rank of each slot, the sort's buffers of the triangle keys
// and ids, then the sorts' temporary storage
ExtractScratch mesh_extract_scratch(long long cap, long long max_tri) { return ExtractScratch{cap, cap, max_tri}; }

cudaError_t launch_mesh_extract(const LrfMeshTable& t, float* xyz, int* faces, long long* counts, void* scratch,
                                cudaStream_t stream) {
  ExtractScratch x = mesh_extract_scratch(t.capacity, t.max_triangles);
  cudaError_t e = x.carve(scratch);
  if (e != cudaSuccess) return e;
  const KeySlotSort &edges = x.pairs[0], &tris = x.pairs[1];
  const unsigned edge_ctas = item_ctas(t.capacity, MC_THREADS), tri_ctas = item_ctas(t.max_triangles, MC_THREADS);
  edge_keys_kernel<<<edge_ctas, MC_THREADS, 0, stream>>>(t, edges.keys(), edges.slots());
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = x.pairs[0].sort(t.capacity, x.temp, x.temp_bytes, stream)) != cudaSuccess) return e;
  vertex_write_kernel<<<edge_ctas, MC_THREADS, 0, stream>>>(t, edges.keys(), edges.slots(), xyz, x.index, counts);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  tri_keys_kernel<<<tri_ctas, MC_THREADS, 0, stream>>>(t, tris.keys(), tris.slots());
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = x.pairs[1].sort(t.max_triangles, x.temp, x.temp_bytes, stream)) != cudaSuccess) return e;
  face_write_kernel<<<tri_ctas, MC_THREADS, 0, stream>>>(t, tris.keys(), tris.slots(), x.index, faces, counts);
  return cudaGetLastError();
}

cudaError_t launch_mesh_normals(const MeshSceneDev& S, const float* xyz, long long n, float* normals, int* owner,
                                cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  mesh_normals_kernel<<<item_ctas(n, MC_THREADS), MC_THREADS, 0, stream>>>(S, xyz, n, normals, owner);
  return cudaGetLastError();
}

}  // namespace lrf
