// mesh.cuh -- marching cubes over a density grid sigma [nx, ny, nz] (C order, k fastest) on the points (xs[i], ys[j], zs[k]):
// the classic Lorensen-Cline cases with Paul Bourke's public-domain 256-entry triangle table, as an indexed mesh.
//
//   * a grid point is inside when sigma > iso (a NaN compares false: outside); cube case bit v is set when corner v is NOT
//     inside (Bourke's `val < iso` with the comparison complemented, so that NaN and sigma == iso are outside);
//   * one vertex per grid edge whose two points differ in inside / outside.  Vertex ids run in grid-point C order, then axis
//     x, y, z, so the cells that share an edge share its vertex;
//   * the vertex on the edge from point a (the lower index) to b along axis ax: t = (iso - s_a) / (s_b - s_a) and
//     c = c_a + t (c_b - c_a), unfused, in that order; the other two coordinates are the grid's own;
//   * faces in cell C order, then table order, wound so that their normals point toward decreasing density.
//
// Two calls, the outputs sized in between by the caller (nerf_b200_marching_cubes_count / _emit): mc_count_kernel writes per
// grid point (vertices on its three edges, triangles of the cell it is the lowest corner of), three deterministic integer scan
// kernels (tiles, the tile sums, the add) turn those into exclusive offsets in place, and mc_emit_kernel writes vertices and
// faces from the offsets.  No atomics: the same sigma gives the same mesh bits on every run.
#pragma once
#include "common.cuh"

namespace nb {

// The exact (FP32) density grid runs mlp_simt_kernel on slabs of the grid: the slab's points [M, 3], row r = point m0 + r in
// C order, copied from the axes without arithmetic (as torch.meshgrid(xs, ys, zs, indexing='ij') builds them) ...
__global__ void __launch_bounds__(256) grid_pts_kernel(const float* __restrict__ xs, const float* __restrict__ ys, const float* __restrict__ zs,
                                                       int ny, int nz, long long m0, long long M, float* __restrict__ pts) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= M) return;
  const long long m = m0 + r, n = m / nz;
  pts[3 * r] = xs[n / ny]; pts[3 * r + 1] = ys[n % ny]; pts[3 * r + 2] = zs[m - n * nz];
}
// ... and the sigma column of its raw rows
__global__ void __launch_bounds__(256) raw_sigma_kernel(const float* __restrict__ raw, long long M, float* __restrict__ sigma) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < M) sigma[r] = raw[4 * r + 3];
}

// corner v of a cell: offset (v & 1) ^ ((v >> 1) & 1) in x, (v >> 1) & 1 in y, v >> 2 in z (Bourke's numbering)
__host__ __device__ constexpr int mc_corner_dx(int v) { return (v & 1) ^ ((v >> 1) & 1); }
__host__ __device__ constexpr int mc_corner_dy(int v) { return (v >> 1) & 1; }
__host__ __device__ constexpr int mc_corner_dz(int v) { return v >> 2; }
// cube edge e -> (lower corner's offset dx, dy, dz, axis 0/1/2): edges 0-3 ring z = 0, 4-7 ring z = 1, 8-11 the z edges
__constant__ const signed char mc_edge_of[12][4] = {
  {0, 0, 0, 0}, {1, 0, 0, 1}, {0, 1, 0, 0}, {0, 0, 0, 1}, {0, 0, 1, 0}, {1, 0, 1, 1},
  {0, 1, 1, 0}, {0, 0, 1, 1}, {0, 0, 0, 2}, {1, 0, 0, 2}, {1, 1, 0, 2}, {0, 1, 0, 2}};

// Paul Bourke's triangle table ("Polygonising a scalar field", public domain): per case, up to five triangles as cube edges,
// -1 terminated.  tests/mc_emul.py reads this table from this file.
__constant__ const signed char mc_tri_table[256][16] = {
  {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 1, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 8, 3, 9, 8, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 3, 1, 2, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {9, 2, 10, 0, 2, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {2, 8, 3, 2, 10, 8, 10, 9, 8, -1, -1, -1, -1, -1, -1, -1},
  {3, 11, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 11, 2, 8, 11, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 9, 0, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 11, 2, 1, 9, 11, 9, 8, 11, -1, -1, -1, -1, -1, -1, -1},
  {3, 10, 1, 11, 10, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 10, 1, 0, 8, 10, 8, 11, 10, -1, -1, -1, -1, -1, -1, -1},
  {3, 9, 0, 3, 11, 9, 11, 10, 9, -1, -1, -1, -1, -1, -1, -1},
  {9, 8, 10, 10, 8, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 3, 0, 7, 3, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 1, 9, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 1, 9, 4, 7, 1, 7, 3, 1, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 10, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {3, 4, 7, 3, 0, 4, 1, 2, 10, -1, -1, -1, -1, -1, -1, -1},
  {9, 2, 10, 9, 0, 2, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1},
  {2, 10, 9, 2, 9, 7, 2, 7, 3, 7, 9, 4, -1, -1, -1, -1},
  {8, 4, 7, 3, 11, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {11, 4, 7, 11, 2, 4, 2, 0, 4, -1, -1, -1, -1, -1, -1, -1},
  {9, 0, 1, 8, 4, 7, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1},
  {4, 7, 11, 9, 4, 11, 9, 11, 2, 9, 2, 1, -1, -1, -1, -1},
  {3, 10, 1, 3, 11, 10, 7, 8, 4, -1, -1, -1, -1, -1, -1, -1},
  {1, 11, 10, 1, 4, 11, 1, 0, 4, 7, 11, 4, -1, -1, -1, -1},
  {4, 7, 8, 9, 0, 11, 9, 11, 10, 11, 0, 3, -1, -1, -1, -1},
  {4, 7, 11, 4, 11, 9, 9, 11, 10, -1, -1, -1, -1, -1, -1, -1},
  {9, 5, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {9, 5, 4, 0, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 5, 4, 1, 5, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {8, 5, 4, 8, 3, 5, 3, 1, 5, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 10, 9, 5, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {3, 0, 8, 1, 2, 10, 4, 9, 5, -1, -1, -1, -1, -1, -1, -1},
  {5, 2, 10, 5, 4, 2, 4, 0, 2, -1, -1, -1, -1, -1, -1, -1},
  {2, 10, 5, 3, 2, 5, 3, 5, 4, 3, 4, 8, -1, -1, -1, -1},
  {9, 5, 4, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 11, 2, 0, 8, 11, 4, 9, 5, -1, -1, -1, -1, -1, -1, -1},
  {0, 5, 4, 0, 1, 5, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1},
  {2, 1, 5, 2, 5, 8, 2, 8, 11, 4, 8, 5, -1, -1, -1, -1},
  {10, 3, 11, 10, 1, 3, 9, 5, 4, -1, -1, -1, -1, -1, -1, -1},
  {4, 9, 5, 0, 8, 1, 8, 10, 1, 8, 11, 10, -1, -1, -1, -1},
  {5, 4, 0, 5, 0, 11, 5, 11, 10, 11, 0, 3, -1, -1, -1, -1},
  {5, 4, 8, 5, 8, 10, 10, 8, 11, -1, -1, -1, -1, -1, -1, -1},
  {9, 7, 8, 5, 7, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {9, 3, 0, 9, 5, 3, 5, 7, 3, -1, -1, -1, -1, -1, -1, -1},
  {0, 7, 8, 0, 1, 7, 1, 5, 7, -1, -1, -1, -1, -1, -1, -1},
  {1, 5, 3, 3, 5, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {9, 7, 8, 9, 5, 7, 10, 1, 2, -1, -1, -1, -1, -1, -1, -1},
  {10, 1, 2, 9, 5, 0, 5, 3, 0, 5, 7, 3, -1, -1, -1, -1},
  {8, 0, 2, 8, 2, 5, 8, 5, 7, 10, 5, 2, -1, -1, -1, -1},
  {2, 10, 5, 2, 5, 3, 3, 5, 7, -1, -1, -1, -1, -1, -1, -1},
  {7, 9, 5, 7, 8, 9, 3, 11, 2, -1, -1, -1, -1, -1, -1, -1},
  {9, 5, 7, 9, 7, 2, 9, 2, 0, 2, 7, 11, -1, -1, -1, -1},
  {2, 3, 11, 0, 1, 8, 1, 7, 8, 1, 5, 7, -1, -1, -1, -1},
  {11, 2, 1, 11, 1, 7, 7, 1, 5, -1, -1, -1, -1, -1, -1, -1},
  {9, 5, 8, 8, 5, 7, 10, 1, 3, 10, 3, 11, -1, -1, -1, -1},
  {5, 7, 0, 5, 0, 9, 7, 11, 0, 1, 0, 10, 11, 10, 0, -1},
  {11, 10, 0, 11, 0, 3, 10, 5, 0, 8, 0, 7, 5, 7, 0, -1},
  {11, 10, 5, 7, 11, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {10, 6, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 3, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {9, 0, 1, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 8, 3, 1, 9, 8, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1},
  {1, 6, 5, 2, 6, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 6, 5, 1, 2, 6, 3, 0, 8, -1, -1, -1, -1, -1, -1, -1},
  {9, 6, 5, 9, 0, 6, 0, 2, 6, -1, -1, -1, -1, -1, -1, -1},
  {5, 9, 8, 5, 8, 2, 5, 2, 6, 3, 2, 8, -1, -1, -1, -1},
  {2, 3, 11, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {11, 0, 8, 11, 2, 0, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1},
  {0, 1, 9, 2, 3, 11, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1},
  {5, 10, 6, 1, 9, 2, 9, 11, 2, 9, 8, 11, -1, -1, -1, -1},
  {6, 3, 11, 6, 5, 3, 5, 1, 3, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 11, 0, 11, 5, 0, 5, 1, 5, 11, 6, -1, -1, -1, -1},
  {3, 11, 6, 0, 3, 6, 0, 6, 5, 0, 5, 9, -1, -1, -1, -1},
  {6, 5, 9, 6, 9, 11, 11, 9, 8, -1, -1, -1, -1, -1, -1, -1},
  {5, 10, 6, 4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 3, 0, 4, 7, 3, 6, 5, 10, -1, -1, -1, -1, -1, -1, -1},
  {1, 9, 0, 5, 10, 6, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1},
  {10, 6, 5, 1, 9, 7, 1, 7, 3, 7, 9, 4, -1, -1, -1, -1},
  {6, 1, 2, 6, 5, 1, 4, 7, 8, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 5, 5, 2, 6, 3, 0, 4, 3, 4, 7, -1, -1, -1, -1},
  {8, 4, 7, 9, 0, 5, 0, 6, 5, 0, 2, 6, -1, -1, -1, -1},
  {7, 3, 9, 7, 9, 4, 3, 2, 9, 5, 9, 6, 2, 6, 9, -1},
  {3, 11, 2, 7, 8, 4, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1},
  {5, 10, 6, 4, 7, 2, 4, 2, 0, 2, 7, 11, -1, -1, -1, -1},
  {0, 1, 9, 4, 7, 8, 2, 3, 11, 5, 10, 6, -1, -1, -1, -1},
  {9, 2, 1, 9, 11, 2, 9, 4, 11, 7, 11, 4, 5, 10, 6, -1},
  {8, 4, 7, 3, 11, 5, 3, 5, 1, 5, 11, 6, -1, -1, -1, -1},
  {5, 1, 11, 5, 11, 6, 1, 0, 11, 7, 11, 4, 0, 4, 11, -1},
  {0, 5, 9, 0, 6, 5, 0, 3, 6, 11, 6, 3, 8, 4, 7, -1},
  {6, 5, 9, 6, 9, 11, 4, 7, 9, 7, 11, 9, -1, -1, -1, -1},
  {10, 4, 9, 6, 4, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 10, 6, 4, 9, 10, 0, 8, 3, -1, -1, -1, -1, -1, -1, -1},
  {10, 0, 1, 10, 6, 0, 6, 4, 0, -1, -1, -1, -1, -1, -1, -1},
  {8, 3, 1, 8, 1, 6, 8, 6, 4, 6, 1, 10, -1, -1, -1, -1},
  {1, 4, 9, 1, 2, 4, 2, 6, 4, -1, -1, -1, -1, -1, -1, -1},
  {3, 0, 8, 1, 2, 9, 2, 4, 9, 2, 6, 4, -1, -1, -1, -1},
  {0, 2, 4, 4, 2, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {8, 3, 2, 8, 2, 4, 4, 2, 6, -1, -1, -1, -1, -1, -1, -1},
  {10, 4, 9, 10, 6, 4, 11, 2, 3, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 2, 2, 8, 11, 4, 9, 10, 4, 10, 6, -1, -1, -1, -1},
  {3, 11, 2, 0, 1, 6, 0, 6, 4, 6, 1, 10, -1, -1, -1, -1},
  {6, 4, 1, 6, 1, 10, 4, 8, 1, 2, 1, 11, 8, 11, 1, -1},
  {9, 6, 4, 9, 3, 6, 9, 1, 3, 11, 6, 3, -1, -1, -1, -1},
  {8, 11, 1, 8, 1, 0, 11, 6, 1, 9, 1, 4, 6, 4, 1, -1},
  {3, 11, 6, 3, 6, 0, 0, 6, 4, -1, -1, -1, -1, -1, -1, -1},
  {6, 4, 8, 11, 6, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {7, 10, 6, 7, 8, 10, 8, 9, 10, -1, -1, -1, -1, -1, -1, -1},
  {0, 7, 3, 0, 10, 7, 0, 9, 10, 6, 7, 10, -1, -1, -1, -1},
  {10, 6, 7, 1, 10, 7, 1, 7, 8, 1, 8, 0, -1, -1, -1, -1},
  {10, 6, 7, 10, 7, 1, 1, 7, 3, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 6, 1, 6, 8, 1, 8, 9, 8, 6, 7, -1, -1, -1, -1},
  {2, 6, 9, 2, 9, 1, 6, 7, 9, 0, 9, 3, 7, 3, 9, -1},
  {7, 8, 0, 7, 0, 6, 6, 0, 2, -1, -1, -1, -1, -1, -1, -1},
  {7, 3, 2, 6, 7, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {2, 3, 11, 10, 6, 8, 10, 8, 9, 8, 6, 7, -1, -1, -1, -1},
  {2, 0, 7, 2, 7, 11, 0, 9, 7, 6, 7, 10, 9, 10, 7, -1},
  {1, 8, 0, 1, 7, 8, 1, 10, 7, 6, 7, 10, 2, 3, 11, -1},
  {11, 2, 1, 11, 1, 7, 10, 6, 1, 6, 7, 1, -1, -1, -1, -1},
  {8, 9, 6, 8, 6, 7, 9, 1, 6, 11, 6, 3, 1, 3, 6, -1},
  {0, 9, 1, 11, 6, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {7, 8, 0, 7, 0, 6, 3, 11, 0, 11, 6, 0, -1, -1, -1, -1},
  {7, 11, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {7, 6, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {3, 0, 8, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 1, 9, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {8, 1, 9, 8, 3, 1, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1},
  {10, 1, 2, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 10, 3, 0, 8, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1},
  {2, 9, 0, 2, 10, 9, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1},
  {6, 11, 7, 2, 10, 3, 10, 8, 3, 10, 9, 8, -1, -1, -1, -1},
  {7, 2, 3, 6, 2, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {7, 0, 8, 7, 6, 0, 6, 2, 0, -1, -1, -1, -1, -1, -1, -1},
  {2, 7, 6, 2, 3, 7, 0, 1, 9, -1, -1, -1, -1, -1, -1, -1},
  {1, 6, 2, 1, 8, 6, 1, 9, 8, 8, 7, 6, -1, -1, -1, -1},
  {10, 7, 6, 10, 1, 7, 1, 3, 7, -1, -1, -1, -1, -1, -1, -1},
  {10, 7, 6, 1, 7, 10, 1, 8, 7, 1, 0, 8, -1, -1, -1, -1},
  {0, 3, 7, 0, 7, 10, 0, 10, 9, 6, 10, 7, -1, -1, -1, -1},
  {7, 6, 10, 7, 10, 8, 8, 10, 9, -1, -1, -1, -1, -1, -1, -1},
  {6, 8, 4, 11, 8, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {3, 6, 11, 3, 0, 6, 0, 4, 6, -1, -1, -1, -1, -1, -1, -1},
  {8, 6, 11, 8, 4, 6, 9, 0, 1, -1, -1, -1, -1, -1, -1, -1},
  {9, 4, 6, 9, 6, 3, 9, 3, 1, 11, 3, 6, -1, -1, -1, -1},
  {6, 8, 4, 6, 11, 8, 2, 10, 1, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 10, 3, 0, 11, 0, 6, 11, 0, 4, 6, -1, -1, -1, -1},
  {4, 11, 8, 4, 6, 11, 0, 2, 9, 2, 10, 9, -1, -1, -1, -1},
  {10, 9, 3, 10, 3, 2, 9, 4, 3, 11, 3, 6, 4, 6, 3, -1},
  {8, 2, 3, 8, 4, 2, 4, 6, 2, -1, -1, -1, -1, -1, -1, -1},
  {0, 4, 2, 4, 6, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 9, 0, 2, 3, 4, 2, 4, 6, 4, 3, 8, -1, -1, -1, -1},
  {1, 9, 4, 1, 4, 2, 2, 4, 6, -1, -1, -1, -1, -1, -1, -1},
  {8, 1, 3, 8, 6, 1, 8, 4, 6, 6, 10, 1, -1, -1, -1, -1},
  {10, 1, 0, 10, 0, 6, 6, 0, 4, -1, -1, -1, -1, -1, -1, -1},
  {4, 6, 3, 4, 3, 8, 6, 10, 3, 0, 3, 9, 10, 9, 3, -1},
  {10, 9, 4, 6, 10, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 9, 5, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 3, 4, 9, 5, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1},
  {5, 0, 1, 5, 4, 0, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1},
  {11, 7, 6, 8, 3, 4, 3, 5, 4, 3, 1, 5, -1, -1, -1, -1},
  {9, 5, 4, 10, 1, 2, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1},
  {6, 11, 7, 1, 2, 10, 0, 8, 3, 4, 9, 5, -1, -1, -1, -1},
  {7, 6, 11, 5, 4, 10, 4, 2, 10, 4, 0, 2, -1, -1, -1, -1},
  {3, 4, 8, 3, 5, 4, 3, 2, 5, 10, 5, 2, 11, 7, 6, -1},
  {7, 2, 3, 7, 6, 2, 5, 4, 9, -1, -1, -1, -1, -1, -1, -1},
  {9, 5, 4, 0, 8, 6, 0, 6, 2, 6, 8, 7, -1, -1, -1, -1},
  {3, 6, 2, 3, 7, 6, 1, 5, 0, 5, 4, 0, -1, -1, -1, -1},
  {6, 2, 8, 6, 8, 7, 2, 1, 8, 4, 8, 5, 1, 5, 8, -1},
  {9, 5, 4, 10, 1, 6, 1, 7, 6, 1, 3, 7, -1, -1, -1, -1},
  {1, 6, 10, 1, 7, 6, 1, 0, 7, 8, 7, 0, 9, 5, 4, -1},
  {4, 0, 10, 4, 10, 5, 0, 3, 10, 6, 10, 7, 3, 7, 10, -1},
  {7, 6, 10, 7, 10, 8, 5, 4, 10, 4, 8, 10, -1, -1, -1, -1},
  {6, 9, 5, 6, 11, 9, 11, 8, 9, -1, -1, -1, -1, -1, -1, -1},
  {3, 6, 11, 0, 6, 3, 0, 5, 6, 0, 9, 5, -1, -1, -1, -1},
  {0, 11, 8, 0, 5, 11, 0, 1, 5, 5, 6, 11, -1, -1, -1, -1},
  {6, 11, 3, 6, 3, 5, 5, 3, 1, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 10, 9, 5, 11, 9, 11, 8, 11, 5, 6, -1, -1, -1, -1},
  {0, 11, 3, 0, 6, 11, 0, 9, 6, 5, 6, 9, 1, 2, 10, -1},
  {11, 8, 5, 11, 5, 6, 8, 0, 5, 10, 5, 2, 0, 2, 5, -1},
  {6, 11, 3, 6, 3, 5, 2, 10, 3, 10, 5, 3, -1, -1, -1, -1},
  {5, 8, 9, 5, 2, 8, 5, 6, 2, 3, 8, 2, -1, -1, -1, -1},
  {9, 5, 6, 9, 6, 0, 0, 6, 2, -1, -1, -1, -1, -1, -1, -1},
  {1, 5, 8, 1, 8, 0, 5, 6, 8, 3, 8, 2, 6, 2, 8, -1},
  {1, 5, 6, 2, 1, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 3, 6, 1, 6, 10, 3, 8, 6, 5, 6, 9, 8, 9, 6, -1},
  {10, 1, 0, 10, 0, 6, 9, 5, 0, 5, 6, 0, -1, -1, -1, -1},
  {0, 3, 8, 5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {10, 5, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {11, 5, 10, 7, 5, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {11, 5, 10, 11, 7, 5, 8, 3, 0, -1, -1, -1, -1, -1, -1, -1},
  {5, 11, 7, 5, 10, 11, 1, 9, 0, -1, -1, -1, -1, -1, -1, -1},
  {10, 7, 5, 10, 11, 7, 9, 8, 1, 8, 3, 1, -1, -1, -1, -1},
  {11, 1, 2, 11, 7, 1, 7, 5, 1, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 3, 1, 2, 7, 1, 7, 5, 7, 2, 11, -1, -1, -1, -1},
  {9, 7, 5, 9, 2, 7, 9, 0, 2, 2, 11, 7, -1, -1, -1, -1},
  {7, 5, 2, 7, 2, 11, 5, 9, 2, 3, 2, 8, 9, 8, 2, -1},
  {2, 5, 10, 2, 3, 5, 3, 7, 5, -1, -1, -1, -1, -1, -1, -1},
  {8, 2, 0, 8, 5, 2, 8, 7, 5, 10, 2, 5, -1, -1, -1, -1},
  {9, 0, 1, 5, 10, 3, 5, 3, 7, 3, 10, 2, -1, -1, -1, -1},
  {9, 8, 2, 9, 2, 1, 8, 7, 2, 10, 2, 5, 7, 5, 2, -1},
  {1, 3, 5, 3, 7, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 7, 0, 7, 1, 1, 7, 5, -1, -1, -1, -1, -1, -1, -1},
  {9, 0, 3, 9, 3, 5, 5, 3, 7, -1, -1, -1, -1, -1, -1, -1},
  {9, 8, 7, 5, 9, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {5, 8, 4, 5, 10, 8, 10, 11, 8, -1, -1, -1, -1, -1, -1, -1},
  {5, 0, 4, 5, 11, 0, 5, 10, 11, 11, 3, 0, -1, -1, -1, -1},
  {0, 1, 9, 8, 4, 10, 8, 10, 11, 10, 4, 5, -1, -1, -1, -1},
  {10, 11, 4, 10, 4, 5, 11, 3, 4, 9, 4, 1, 3, 1, 4, -1},
  {2, 5, 1, 2, 8, 5, 2, 11, 8, 4, 5, 8, -1, -1, -1, -1},
  {0, 4, 11, 0, 11, 3, 4, 5, 11, 2, 11, 1, 5, 1, 11, -1},
  {0, 2, 5, 0, 5, 9, 2, 11, 5, 4, 5, 8, 11, 8, 5, -1},
  {9, 4, 5, 2, 11, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {2, 5, 10, 3, 5, 2, 3, 4, 5, 3, 8, 4, -1, -1, -1, -1},
  {5, 10, 2, 5, 2, 4, 4, 2, 0, -1, -1, -1, -1, -1, -1, -1},
  {3, 10, 2, 3, 5, 10, 3, 8, 5, 4, 5, 8, 0, 1, 9, -1},
  {5, 10, 2, 5, 2, 4, 1, 9, 2, 9, 4, 2, -1, -1, -1, -1},
  {8, 4, 5, 8, 5, 3, 3, 5, 1, -1, -1, -1, -1, -1, -1, -1},
  {0, 4, 5, 1, 0, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {8, 4, 5, 8, 5, 3, 9, 0, 5, 0, 3, 5, -1, -1, -1, -1},
  {9, 4, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 11, 7, 4, 9, 11, 9, 10, 11, -1, -1, -1, -1, -1, -1, -1},
  {0, 8, 3, 4, 9, 7, 9, 11, 7, 9, 10, 11, -1, -1, -1, -1},
  {1, 10, 11, 1, 11, 4, 1, 4, 0, 7, 4, 11, -1, -1, -1, -1},
  {3, 1, 4, 3, 4, 8, 1, 10, 4, 7, 4, 11, 10, 11, 4, -1},
  {4, 11, 7, 9, 11, 4, 9, 2, 11, 9, 1, 2, -1, -1, -1, -1},
  {9, 7, 4, 9, 11, 7, 9, 1, 11, 2, 11, 1, 0, 8, 3, -1},
  {11, 7, 4, 11, 4, 2, 2, 4, 0, -1, -1, -1, -1, -1, -1, -1},
  {11, 7, 4, 11, 4, 2, 8, 3, 4, 3, 2, 4, -1, -1, -1, -1},
  {2, 9, 10, 2, 7, 9, 2, 3, 7, 7, 4, 9, -1, -1, -1, -1},
  {9, 10, 7, 9, 7, 4, 10, 2, 7, 8, 7, 0, 2, 0, 7, -1},
  {3, 7, 10, 3, 10, 2, 7, 4, 10, 1, 10, 0, 4, 0, 10, -1},
  {1, 10, 2, 8, 7, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 9, 1, 4, 1, 7, 7, 1, 3, -1, -1, -1, -1, -1, -1, -1},
  {4, 9, 1, 4, 1, 7, 0, 8, 1, 8, 7, 1, -1, -1, -1, -1},
  {4, 0, 3, 7, 4, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {4, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {9, 10, 8, 10, 11, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {3, 0, 9, 3, 9, 11, 11, 9, 10, -1, -1, -1, -1, -1, -1, -1},
  {0, 1, 10, 0, 10, 8, 8, 10, 11, -1, -1, -1, -1, -1, -1, -1},
  {3, 1, 10, 11, 3, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 2, 11, 1, 11, 9, 9, 11, 8, -1, -1, -1, -1, -1, -1, -1},
  {3, 0, 9, 3, 9, 11, 1, 2, 9, 2, 11, 9, -1, -1, -1, -1},
  {0, 2, 11, 8, 0, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {3, 2, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {2, 3, 8, 2, 8, 10, 10, 8, 9, -1, -1, -1, -1, -1, -1, -1},
  {9, 10, 2, 0, 9, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {2, 3, 8, 2, 8, 10, 0, 1, 8, 1, 10, 8, -1, -1, -1, -1},
  {1, 10, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {1, 3, 8, 9, 1, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 9, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {0, 3, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
  {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1}};

// scan tiles: 1024 threads x 4 consecutive items
constexpr int MC_SCAN_THREADS = 1024, MC_SCAN_ITEMS = 4, MC_SCAN_TILE = MC_SCAN_THREADS * MC_SCAN_ITEMS;
// workspace header (before the per-point offsets): V, F and the grid and iso the counts belong to
struct McHeader { long long V, F; int nx, ny, nz; float iso; };
constexpr size_t MC_HEADER_BYTES = 256;

__device__ __forceinline__ bool mc_inside(float s, float iso) { return s > iso; }

__device__ __forceinline__ int mc_case(const float* __restrict__ sigma, long long p, long long sx, long long sy, float iso) {
  int ci = 0;
#pragma unroll
  for (int v = 0; v < 8; ++v)
    if (!mc_inside(sigma[p + mc_corner_dx(v) * sx + mc_corner_dy(v) * sy + mc_corner_dz(v)], iso)) ci |= 1 << v;
  return ci;
}
__device__ __forceinline__ int mc_ntri(int ci) {
  int n = 0;
  while (n < 5 && mc_tri_table[ci][3 * n] >= 0) ++n;
  return n;
}

// per grid point p = (i, j, k): (vertices on its edges toward +x, +y, +z, triangles of the cell whose lowest corner it is)
__global__ void __launch_bounds__(256) mc_count_kernel(const float* __restrict__ sigma, int nx, int ny, int nz, float iso, int2* __restrict__ cnt) {
  const long long P = (long long)nx * ny * nz, p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const long long sy = nz, sx = (long long)ny * nz;
  const int k = (int)(p % nz), j = (int)((p / nz) % ny), i = (int)(p / sx);
  const bool a = mc_inside(sigma[p], iso);
  int nv = 0, nt = 0;
  if (i + 1 < nx) nv += a != mc_inside(sigma[p + sx], iso);
  if (j + 1 < ny) nv += a != mc_inside(sigma[p + sy], iso);
  if (k + 1 < nz) nv += a != mc_inside(sigma[p + 1], iso);
  if (i + 1 < nx && j + 1 < ny && k + 1 < nz) nt = mc_ntri(mc_case(sigma, p, sx, sy, iso));
  cnt[p] = make_int2(nv, nt);
}

// exclusive scan of one tile of `v` in place; the tile's total -> tsum[tile]
__global__ void __launch_bounds__(MC_SCAN_THREADS) mc_scan_tiles_kernel(int2* __restrict__ v, long long n, int2* __restrict__ tsum) {
  __shared__ int2 s_warp[MC_SCAN_THREADS / 32];
  const long long base = (long long)blockIdx.x * MC_SCAN_TILE + (long long)threadIdx.x * MC_SCAN_ITEMS;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int2 it[MC_SCAN_ITEMS], tot = make_int2(0, 0);
#pragma unroll
  for (int q = 0; q < MC_SCAN_ITEMS; ++q) {
    it[q] = base + q < n ? v[base + q] : make_int2(0, 0);
    const int2 c = it[q];
    it[q] = tot;                                         // exclusive within the thread
    tot.x += c.x; tot.y += c.y;
  }
  int2 inc = tot;                                        // inclusive over the warp's threads
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int x = __shfl_up_sync(0xffffffffu, inc.x, o), y = __shfl_up_sync(0xffffffffu, inc.y, o);
    if (lane >= o) { inc.x += x; inc.y += y; }
  }
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int2 w = s_warp[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int x = __shfl_up_sync(0xffffffffu, wi.x, o), y = __shfl_up_sync(0xffffffffu, wi.y, o);
      if (lane >= o) { wi.x += x; wi.y += y; }
    }
    s_warp[lane] = make_int2(wi.x - w.x, wi.y - w.y);   // exclusive over the warps
    if (lane == 31) tsum[blockIdx.x] = wi;
  }
  __syncthreads();
  const int2 off = make_int2(s_warp[wid].x + inc.x - tot.x, s_warp[wid].y + inc.y - tot.y);
#pragma unroll
  for (int q = 0; q < MC_SCAN_ITEMS; ++q)
    if (base + q < n) v[base + q] = make_int2(off.x + it[q].x, off.y + it[q].y);
}

// exclusive scan of the nt tile sums in place (one block, 1024 sums at a time with a carry); the totals -> counts and the header
__global__ void __launch_bounds__(MC_SCAN_THREADS) mc_scan_sums_kernel(int2* __restrict__ tsum, int nt, long long* __restrict__ counts,
                                                                   McHeader* __restrict__ hdr, McHeader grid) {
  __shared__ int2 s_warp[MC_SCAN_THREADS / 32];
  __shared__ int2 s_tot;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long cx = 0, cy = 0;                              // carry (the caller checks that the totals fit in 31 bits)
  for (int b0 = 0; b0 < nt; b0 += MC_SCAN_THREADS) {
    const int b = b0 + threadIdx.x;
    const int2 c = b < nt ? tsum[b] : make_int2(0, 0);
    int2 inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int x = __shfl_up_sync(0xffffffffu, inc.x, o), y = __shfl_up_sync(0xffffffffu, inc.y, o);
      if (lane >= o) { inc.x += x; inc.y += y; }
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      const int2 w = s_warp[lane];
      int2 wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, wi.x, o), y = __shfl_up_sync(0xffffffffu, wi.y, o);
        if (lane >= o) { wi.x += x; wi.y += y; }
      }
      s_warp[lane] = make_int2(wi.x - w.x, wi.y - w.y);
      if (lane == 31) s_tot = wi;
    }
    __syncthreads();
    if (b < nt) tsum[b] = make_int2((int)(cx + s_warp[wid].x + inc.x - c.x), (int)(cy + s_warp[wid].y + inc.y - c.y));
    cx += s_tot.x; cy += s_tot.y;
    __syncthreads();                                     // s_warp and s_tot are rewritten by the next 1024 sums
  }
  if (threadIdx.x == 0) {
    counts[0] = cx; counts[1] = cy;
    grid.V = cx; grid.F = cy;
    *hdr = grid;
  }
}

// v[i] += tsum[tile of i]: the offsets of the whole grid
__global__ void __launch_bounds__(256) mc_scan_add_kernel(int2* __restrict__ v, long long n, const int2* __restrict__ tsum) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int2 t = tsum[i / MC_SCAN_TILE], a = v[i];
  v[i] = make_int2(a.x + t.x, a.y + t.y);
}

// edge (point q = (qi, qj, qk), axis ax) has a vertex: both ends exist and differ in inside / outside
__device__ __forceinline__ bool mc_active(const float* __restrict__ sigma, int qi, int qj, int qk, int ax, int nx, int ny, int nz, float iso) {
  const long long sy = nz, sx = (long long)ny * nz, q = qi * sx + qj * sy + qk;
  if (ax == 0) return qi + 1 < nx && mc_inside(sigma[q], iso) != mc_inside(sigma[q + sx], iso);
  if (ax == 1) return qj + 1 < ny && mc_inside(sigma[q], iso) != mc_inside(sigma[q + sy], iso);
  return qk + 1 < nz && mc_inside(sigma[q], iso) != mc_inside(sigma[q + 1], iso);
}
// the position along the edge from a to b: t = (iso - s_a) / (s_b - s_a), c = c_a + t (c_b - c_a), unfused
__device__ __forceinline__ float mc_lerp(float sa, float sb, float ca, float cb, float iso) {
  const float t = __fdiv_rn(__fsub_rn(iso, sa), __fsub_rn(sb, sa));
  return __fadd_rn(ca, __fmul_rn(t, __fsub_rn(cb, ca)));
}

// per grid point: the vertices of its edges, then the faces of its cell (off: the scanned offsets of mc_count_kernel's counts)
__global__ void __launch_bounds__(256) mc_emit_kernel(const float* __restrict__ sigma, const float* __restrict__ xs, const float* __restrict__ ys,
                                                      const float* __restrict__ zs, int nx, int ny, int nz, float iso,
                                                      const int2* __restrict__ off, float* __restrict__ verts, int* __restrict__ faces) {
  const long long P = (long long)nx * ny * nz, p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const long long sy = nz, sx = (long long)ny * nz;
  const int k = (int)(p % nz), j = (int)((p / nz) % ny), i = (int)(p / sx);
  const float s = sigma[p];
  const bool a = mc_inside(s, iso);
  int vid = off[p].x;
  if (i + 1 < nx) {
    const float sb = sigma[p + sx];
    if (a != mc_inside(sb, iso)) {
      float* o = verts + 3ll * vid++;
      o[0] = mc_lerp(s, sb, xs[i], xs[i + 1], iso); o[1] = ys[j]; o[2] = zs[k];
    }
  }
  if (j + 1 < ny) {
    const float sb = sigma[p + sy];
    if (a != mc_inside(sb, iso)) {
      float* o = verts + 3ll * vid++;
      o[0] = xs[i]; o[1] = mc_lerp(s, sb, ys[j], ys[j + 1], iso); o[2] = zs[k];
    }
  }
  if (k + 1 < nz) {
    const float sb = sigma[p + 1];
    if (a != mc_inside(sb, iso)) {
      float* o = verts + 3ll * vid;
      o[0] = xs[i]; o[1] = ys[j]; o[2] = mc_lerp(s, sb, zs[k], zs[k + 1], iso);
    }
  }
  if (!(i + 1 < nx && j + 1 < ny && k + 1 < nz)) return;
  const int ci = mc_case(sigma, p, sx, sy, iso);
  int* f = faces + 3ll * off[p].y;
  for (int t = 0; t < 5 && mc_tri_table[ci][3 * t] >= 0; ++t) {
    int id[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const signed char* e = mc_edge_of[mc_tri_table[ci][3 * t + c]];
      const int qi = i + e[0], qj = j + e[1], qk = k + e[2], ax = e[3];
      // the edge's vertex id: the point's first id plus its active edges along the axes before ax
      int r = off[(long long)qi * sx + qj * sy + qk].x;
      if (ax > 0) r += mc_active(sigma, qi, qj, qk, 0, nx, ny, nz, iso);
      if (ax > 1) r += mc_active(sigma, qi, qj, qk, 1, nx, ny, nz, iso);
      id[c] = r;
    }
    // with the case bits of the corners NOT inside, the table's own winding puts the normals toward decreasing density
    f[3 * t] = id[0]; f[3 * t + 1] = id[1]; f[3 * t + 2] = id[2];
  }
}

}  // namespace nb
