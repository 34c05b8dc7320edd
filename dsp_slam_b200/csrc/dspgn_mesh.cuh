// Iso-surface of SDF grids on the device: MeshExtractor.extract_mesh_from_code (reconstruct/optimizer.py:214-223) for a
// batch of objects, as dsp_slam_b200/mesh.py's marching tetrahedra computes it, bit for bit.
//
// Grid: object o, lattice vertex (x, y, z) of a dim^3 grid = row (x*dim + y)*dim + z of the object's SDF block (the row
// order of create_voxel_grid, optimizer.py:490-504), spacing h = 2/(dim-1), the level set sdf = 0, inside = sdf < 0.
// Kuhn subdivision: 6 tetrahedra around the 0-6 diagonal of every cube, so every tetrahedron edge runs from a lattice
// vertex `lo` to lo + one of 7 positive offsets (dx, dy, dz) != 0, numbered k = 4dx + 2dy + dz - 1 (z, y, yz, x, xz, xy,
// xyz: increasing flat offset).  mesh.py numbers its vertices by np.unique of (lo, hi) edge keys, i.e. by lo, then k: an
// exclusive scan of the per-lattice-vertex 7-bit masks of the edges that carry a vertex gives exactly those ids.
// An edge carries a vertex when its ends lie on both sides and at least one cube containing it has no NaN corner
// (mesh.py skips a cube with a NaN corner: min / max propagate NaN).
//
// Faces come in four groups -- tetrahedra with 1 corner inside; 3 inside; the first, then the second triangle of the
// 2-inside quads -- each in cube order, then tetrahedron order; a triangle is flipped when its fp64 normal points against
// (mean of the outside corners - mean of the inside corners) and dropped when its squared area is <= 1e-30.
// Passes: k_mesh_cubes (per-cube NaN flag and group counts) -> k_mesh_verts (edge masks) -> integer scans -> one
// read-back of the per-object totals -> k_mesh_emit_verts / k_mesh_emit_faces (or, in a submitted keyframe call, no
// read-back and the *_arena variants below).
// Every fp64 step is an explicit _rn intrinsic: numpy rounds each operation, and the build's --fmad=true must not
// contract them.
#pragma once
#include <cstdint>

namespace dspgn {

constexpr int kMeshMaxDim = 128;
constexpr long long kMeshChunkRows = 1LL << 24;    // grid rows (objects x dim^3) per chunk of a mesh call

struct MeshGrid {
  const float* sdf;     // [n][dim^3]
  int n, dim;
  long long R, C;       // dim^3 lattice vertices, (dim-1)^3 cubes per object
  double h;             // 2 / (dim - 1), fp64 like mesh.py's spacing
};

// cube corners (x, y, z) and the six tetrahedra, as mesh.py's _CORNERS / _TETS
__constant__ int8_t c_mesh_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
__constant__ int8_t c_mesh_tet[6][4] = {{0, 5, 1, 6}, {0, 1, 2, 6}, {0, 2, 3, 6}, {0, 3, 7, 6}, {0, 7, 4, 6}, {0, 4, 5, 6}};
// the triangle corners of each group as (i, j) pairs of the inside-first corner order (mesh.py emit calls)
__constant__ int8_t c_mesh_tri[4][3][2] = {{{0, 1}, {0, 2}, {0, 3}}, {{3, 0}, {3, 1}, {3, 2}},
                                           {{0, 2}, {0, 3}, {1, 3}}, {{0, 2}, {1, 3}, {1, 2}}};

// The query grid of create_voxel_grid(dim) (optimizer.py:490-504, the reference's true-division shear) into the points
// block: object o's rows at o * dim^3, xyz interleaved.
__global__ void k_mesh_grid_points(float* pts, int n, int dim) {
  const long long R = (long long)dim * dim * dim;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  const float fd = (float)dim;
  const float vs = __double2float_rn(__ddiv_rn(2.0, (double)(dim - 1)));
  const float q = __double2float_rn(__ddiv_rn((double)i, (double)dim));
  const float z = (float)(i % dim);
  const float y = fmodf(q, fd);
  const float x = fmodf(__fdiv_rn(q, fd), fd);
  const float p0 = __fadd_rn(__fmul_rn(x, vs), -1.f), p1 = __fadd_rn(__fmul_rn(y, vs), -1.f), p2 = __fadd_rn(__fmul_rn(z, vs), -1.f);
  for (int o = blockIdx.y; o < n; o += gridDim.y) {
    float* p = pts + 3 * ((size_t)o * R + i);
    p[0] = p0; p[1] = p1; p[2] = p2;
  }
}

__device__ __forceinline__ double mesh_sdf(const MeshGrid& g, const float* s, int x, int y, int z) {
  return (double)s[((long long)x * g.dim + y) * g.dim + z];
}

// mesh.py's vertex of the edge lo -> lo + offset k: t = (0 - va) / (vb - va), p = pa + t (pb - pa), pa = index * h (fp64)
__device__ __forceinline__ void mesh_edge_point(const MeshGrid& g, const float* s, int x, int y, int z, int k, double p[3]) {
  const int d[3] = {((k + 1) >> 2) & 1, ((k + 1) >> 1) & 1, (k + 1) & 1};
  const int lo[3] = {x, y, z};
  const double va = mesh_sdf(g, s, x, y, z), vb = mesh_sdf(g, s, x + d[0], y + d[1], z + d[2]);
  const double t = __ddiv_rn(__dsub_rn(0.0, va), __dsub_rn(vb, va));
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double pa = __dmul_rn((double)lo[a], g.h), pb = __dmul_rn((double)(lo[a] + d[a]), g.h);
    p[a] = __dadd_rn(pa, __dmul_rn(t, __dsub_rn(pb, pa)));
  }
}

// One cube's corner values; mesh.py meshes it only when it has no NaN corner and the level set crosses it.
struct MeshCube {
  float v[8];
  bool ok, crossed;
};

__device__ __forceinline__ MeshCube mesh_load_cube(const MeshGrid& g, const float* s, int bx, int by, int bz) {
  MeshCube c;
  bool nan = false, any_in = false, any_out = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    c.v[k] = s[((long long)(bx + c_mesh_corner[k][0]) * g.dim + (by + c_mesh_corner[k][1])) * g.dim + (bz + c_mesh_corner[k][2])];
    nan |= isnan(c.v[k]);
    any_in |= c.v[k] < 0.f;
    any_out |= c.v[k] >= 0.f;
  }
  c.ok = !nan;
  c.crossed = !nan && any_in && any_out;
  return c;
}

// The inside-first corner order of tetrahedron t (a stable partition, like mesh.py's argsort) and its inside count.
struct MeshTet { int8_t c[4]; int cnt; };

__device__ __forceinline__ MeshTet mesh_tet(const MeshCube& cube, int t) {
  MeshTet r;
  int n_in = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) n_in += cube.v[c_mesh_tet[t][j]] < 0.f;
  int a = 0, b = n_in;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int8_t c = c_mesh_tet[t][j];
    if (cube.v[c] < 0.f) r.c[a++] = c; else r.c[b++] = c;
  }
  r.cnt = n_in;
  return r;
}

// the fp64 triangle of group gi of tetrahedron tt, its orientation test and its squared area
struct MeshTri {
  int lo[3][3];   // lattice vertex `lo` of each corner's edge
  int k[3];       // and its offset index
  bool flip, keep;
};

__device__ __forceinline__ MeshTri mesh_tri(const MeshGrid& g, const float* s, int bx, int by, int bz, const MeshTet& tt, int gi) {
  MeshTri T;
  double P[3][3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int ca = tt.c[c_mesh_tri[gi][j][0]], cb = tt.c[c_mesh_tri[gi][j][1]];
    int d[3], l[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int ea = c_mesh_corner[ca][a], eb = c_mesh_corner[cb][a];
      l[a] = min(ea, eb); d[a] = max(ea, eb) - l[a];       // Kuhn edges join comparable corners
    }
    T.lo[j][0] = bx + l[0]; T.lo[j][1] = by + l[1]; T.lo[j][2] = bz + l[2];
    T.k[j] = 4 * d[0] + 2 * d[1] + d[2] - 1;
    mesh_edge_point(g, s, T.lo[j][0], T.lo[j][1], T.lo[j][2], T.k[j], P[j]);
  }
  // mean of the inside / outside corner positions (fp64: sequential sum, then / count)
  double ins[3], outs[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int base = a == 0 ? bx : (a == 1 ? by : bz);
    double si = 0.0, so = 0.0;
    for (int j = 0; j < 4; ++j) {
      const double pj = __dmul_rn((double)(base + c_mesh_corner[tt.c[j]][a]), g.h);
      if (j < tt.cnt) si = (j == 0) ? pj : __dadd_rn(si, pj);
      else so = (j == tt.cnt) ? pj : __dadd_rn(so, pj);
    }
    ins[a] = __ddiv_rn(si, (double)tt.cnt);
    outs[a] = __ddiv_rn(so, (double)(4 - tt.cnt));
  }
  double u[3], w[3], R[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    u[a] = __dsub_rn(P[1][a], P[0][a]);
    w[a] = __dsub_rn(P[2][a], P[0][a]);
    R[a] = __dsub_rn(outs[a], ins[a]);
  }
  const double n0 = __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1]));   // np.cross
  const double n1 = __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2]));
  const double n2 = __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0]));
  const double dot = __dadd_rn(__dadd_rn(__dmul_rn(n0, R[0]), __dmul_rn(n1, R[1])), __dmul_rn(n2, R[2]));
  const double area2 = __dadd_rn(__dadd_rn(__dmul_rn(n0, n0), __dmul_rn(n1, n1)), __dmul_rn(n2, n2));
  T.flip = dot < 0.0;
  T.keep = area2 > 1e-30;
  return T;
}

// pass 1, one thread per cube: NaN-free flag and the kept triangles of each group.
// ok[o][c]; cnt[(o*4 + group)][c]
__global__ void k_mesh_cubes(MeshGrid g, uint8_t* ok, int* cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)g.n * g.C) return;
  const int o = (int)(i / g.C);
  const long long c = i - (long long)o * g.C;
  const int m = g.dim - 1;
  const int bx = (int)(c / ((long long)m * m)), by = (int)((c / m) % m), bz = (int)(c % m);
  const float* s = g.sdf + (size_t)o * g.R;
  const MeshCube cube = mesh_load_cube(g, s, bx, by, bz);
  int n[4] = {0, 0, 0, 0};
  if (cube.crossed) {
    for (int t = 0; t < 6; ++t) {
      const MeshTet tt = mesh_tet(cube, t);
      if (tt.cnt == 0 || tt.cnt == 4) continue;
      const int g0 = tt.cnt == 1 ? 0 : (tt.cnt == 3 ? 1 : 2);
      for (int gi = g0; gi <= (tt.cnt == 2 ? 3 : g0); ++gi) n[gi] += mesh_tri(g, s, bx, by, bz, tt, gi).keep;
    }
  }
  ok[i] = cube.ok;
#pragma unroll
  for (int gi = 0; gi < 4; ++gi) cnt[((size_t)o * 4 + gi) * g.C + c] = n[gi];
}

// pass 2, one thread per lattice vertex: the 7-bit mask of its edges that carry a vertex, and its popcount
__global__ void k_mesh_verts(MeshGrid g, const uint8_t* ok, uint8_t* mask, int* cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)g.n * g.R) return;
  const int o = (int)(i / g.R);
  const long long v = i - (long long)o * g.R;
  const int dm = g.dim, m = dm - 1;
  const int x = (int)(v / ((long long)dm * dm)), y = (int)((v / dm) % dm), z = (int)(v % dm);
  const float* s = g.sdf + (size_t)o * g.R;
  const uint8_t* ok_o = ok + (size_t)o * g.C;
  const bool in_a = s[v] < 0.f;
  unsigned bits = 0;
  for (int k = 0; k < 7; ++k) {
    const int dx = ((k + 1) >> 2) & 1, dy = ((k + 1) >> 1) & 1, dz = (k + 1) & 1;
    if (x + dx >= dm || y + dy >= dm || z + dz >= dm) continue;
    if ((s[((long long)(x + dx) * dm + (y + dy)) * dm + (z + dz)] < 0.f) == in_a) continue;
    // the cubes that contain the edge: base = lo on the axes it runs along, lo - 1 or lo on the others
    bool any = false;
    for (int cx = x - 1 + dx; cx <= x && !any; ++cx)
      for (int cy = y - 1 + dy; cy <= y && !any; ++cy)
        for (int cz = z - 1 + dz; cz <= z && !any; ++cz)
          if (cx >= 0 && cy >= 0 && cz >= 0 && cx < m && cy < m && cz < m) any = ok_o[((long long)cx * m + cy) * m + cz] != 0;
    if (any) bits |= 1u << k;
  }
  mask[i] = (uint8_t)bits;
  cnt[i] = __popc(bits);
}

// the first vertex / face of every object of the chunk (object n: the chunk's totals), from the exclusive scans
__global__ void k_mesh_bases(MeshGrid g, const int* vscan, const int* fscan, int* out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o > g.n) return;
  out[2 * o] = vscan[(size_t)o * g.R];
  out[2 * o + 1] = fscan[(size_t)o * 4 * g.C];
}

// pass 3a, one thread per lattice vertex: its vertices, f32(f32(p) + (-1.0)) as extract_mesh_from_code returns them
__device__ __forceinline__ void mesh_emit_verts(const MeshGrid& g, const uint8_t* mask, const int* vscan, float* verts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)g.n * g.R) return;
  unsigned bits = mask[i];
  if (!bits) return;
  const int o = (int)(i / g.R);
  const long long v = i - (long long)o * g.R;
  const int dm = g.dim;
  const int x = (int)(v / ((long long)dm * dm)), y = (int)((v / dm) % dm), z = (int)(v % dm);
  const float* s = g.sdf + (size_t)o * g.R;
  float* out = verts + 3 * (size_t)vscan[i];
  for (; bits; bits &= bits - 1, out += 3) {
    double p[3];
    mesh_edge_point(g, s, x, y, z, __ffs(bits) - 1, p);
#pragma unroll
    for (int a = 0; a < 3; ++a) out[a] = __double2float_rn(__dadd_rn((double)__double2float_rn(p[a]), -1.0));
  }
}

// pass 3b, one thread per cube: its kept triangles at their place in the object's four groups; indices local to the
// object's vertices
__device__ __forceinline__ void mesh_emit_faces(const MeshGrid& g, const uint8_t* mask, const int* vscan, const int* fscan,
                                                int32_t* faces) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)g.n * g.C) return;
  const int o = (int)(i / g.C);
  const long long c = i - (long long)o * g.C;
  const int m = g.dim - 1, dm = g.dim;
  const int bx = (int)(c / ((long long)m * m)), by = (int)((c / m) % m), bz = (int)(c % m);
  const float* s = g.sdf + (size_t)o * g.R;
  const MeshCube cube = mesh_load_cube(g, s, bx, by, bz);
  if (!cube.crossed) return;
  const size_t vo = (size_t)o * g.R;
  const int v0 = vscan[vo];
  int next[4];
#pragma unroll
  for (int gi = 0; gi < 4; ++gi) next[gi] = fscan[((size_t)o * 4 + gi) * g.C + c];
  for (int t = 0; t < 6; ++t) {
    const MeshTet tt = mesh_tet(cube, t);
    if (tt.cnt == 0 || tt.cnt == 4) continue;
    const int g0 = tt.cnt == 1 ? 0 : (tt.cnt == 3 ? 1 : 2);
    for (int gi = g0; gi <= (tt.cnt == 2 ? 3 : g0); ++gi) {
      const MeshTri T = mesh_tri(g, s, bx, by, bz, tt, gi);
      if (!T.keep) continue;
      int id[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const size_t lv = vo + ((size_t)T.lo[j][0] * dm + T.lo[j][1]) * dm + T.lo[j][2];
        id[j] = vscan[lv] + __popc(mask[lv] & ((1u << T.k[j]) - 1u)) - v0;
      }
      int32_t* f = faces + 3 * (size_t)next[gi]++;
      f[0] = id[0]; f[1] = T.flip ? id[2] : id[1]; f[2] = T.flip ? id[1] : id[2];
    }
  }
}

__global__ void k_mesh_emit_verts(MeshGrid g, const uint8_t* mask, const int* vscan, float* verts) {
  mesh_emit_verts(g, mask, vscan, verts);
}

__global__ void k_mesh_emit_faces(MeshGrid g, const uint8_t* mask, const int* vscan, const int* fscan, int32_t* faces) {
  mesh_emit_faces(g, mask, vscan, fscan, faces);
}

// The emit passes of a submitted keyframe call (dspgn_keyframe_submit), which places its meshes without reading the
// counts back: vertices and faces go into an arena of cap_v vertices | cap_f faces sized on the host beforehand.  When
// the chunk's totals (k_mesh_bases' entry n) do not fit, nothing is written and dspgn_keyframe_wait re-runs
// k_mesh_emit_verts / k_mesh_emit_faces at the exact sizes from the same grids and scans.
__device__ __forceinline__ bool mesh_arena_fits(const int* totals, long long cap_v, long long cap_f) {
  return totals[0] <= cap_v && totals[1] <= cap_f;
}

__global__ void k_mesh_emit_verts_arena(MeshGrid g, const uint8_t* mask, const int* vscan, const int* totals, long long cap_v,
                                        long long cap_f, float* arena) {
  if (!mesh_arena_fits(totals, cap_v, cap_f)) return;
  mesh_emit_verts(g, mask, vscan, arena);
}

__global__ void k_mesh_emit_faces_arena(MeshGrid g, const uint8_t* mask, const int* vscan, const int* fscan,
                                        const int* totals, long long cap_v, long long cap_f, float* arena) {
  if (!mesh_arena_fits(totals, cap_v, cap_f)) return;
  mesh_emit_faces(g, mask, vscan, fscan, reinterpret_cast<int32_t*>(arena + 3 * cap_v));
}

}  // namespace dspgn
