// vxx_layout.h -- how the warp-per-instance sweep stores the cost-to-go Hessians Vxx.
//
// Vxx_t for t >= 1 is exactly symmetric (the sweep mirrors the lower triangle of V'), so only its
// lower triangle is stored, packed column by column (LAPACK 'L'): column j holds rows j..nx-1.  One
// knot takes vxx_packed_doubles(nx) doubles, nx(nx+1)/2 rounded up to even so that every knot
// starts 16 bytes aligned (bulk copies); the padding double is written as 0.
//   packed array: [batch][N+1][vxx_packed_doubles(nx)]
//   full array:   [batch][nx*nx], column-major
// Physical factor slot 0 is the one block that is not symmetric in general: the unsymmetrised
// Vxx_0 of the reference (and the terminal block when N = 0).  It lives in the full array; the
// packed slot 0 is unused.  The CTA-per-instance and dense kernels keep the plain full layout
// [batch][N+1][nx*nx].
#pragma once

#if defined(__CUDACC__)
#define AB2_VXX_HD __host__ __device__ __forceinline__
#else
#define AB2_VXX_HD inline
#endif

namespace ab2 {

AB2_VXX_HD constexpr int vxx_packed_doubles(int nx) { return (nx * (nx + 1) / 2 + 1) & ~1; }
// first packed entry of column j
AB2_VXX_HD constexpr int vxx_packed_col(int nx, int j) { return j * nx - j * (j - 1) / 2; }
// packed entry of the symmetric block's (i, j), either triangle
AB2_VXX_HD constexpr int vxx_packed_index(int nx, int i, int j) {
  return i >= j ? vxx_packed_col(nx, j) + (i - j) : vxx_packed_col(nx, i) + (j - i);
}
// the block of physical factor slot `slot` is stored in full (the separate [batch][nx*nx] array)
AB2_VXX_HD constexpr bool vxx_slot_is_full(int slot) { return slot == 0; }
// (i, j), i >= j, of packed entry e < nx(nx+1)/2
AB2_VXX_HD void vxx_packed_coords(int nx, int e, int &i, int &j) {
  j = 0;
  while (e >= nx - j) {
    e -= nx - j;
    ++j;
  }
  i = j + e;
}

} // namespace ab2
