// strolle_b200 — ST_OPT_BVH_REFIT: device bake of moved instances and bottom-up refit of the BVH boxes.
//
// The bake restates engine.cu's bake_triangle with the flag-independent x*() primitives of st_math.cuh, in the host's operation
// order, so that the device writes the bits the host would have written (no build flag can contract or approximate it).  The refit
// recomputes every box of the flattened stream (engine.cu BvhBuild::emit) from the baked triangles over the kept topology: leaf runs
// first, then the internal nodes level by level from the deepest one up.  A box is a min/max reduction, so the result does not depend
// on the order the threads run in.
#include "kernels.h"
#include "st_math.cuh"

namespace st {

// Rust's NaN-ignoring f32::min / f32::max (Box::grow), with -0 ordered below +0 so that the reduction is order-independent
ST_DEV float bmin(float a, float b) { if (a != a) return b; if (b != b) return a; return (a < b || (a == b && (fbits(a) >> 31))) ? a : b; }
ST_DEV float bmax(float a, float b) { if (a != a) return b; if (b != b) return a; return (a > b || (a == b && !(fbits(a) >> 31))) ? a : b; }

// aff_mat / aff_point / hnorm of engine.cu, one correctly rounded operation at a time
ST_DEV float3 aff_mat3(const float* m, float3 v) {   // m: x.xyz, y.xyz, z.xyz
    return f3(xadd(xadd(xmul(m[0], v.x), xmul(m[3], v.y)), xmul(m[6], v.z)),
              xadd(xadd(xmul(m[1], v.x), xmul(m[4], v.y)), xmul(m[7], v.z)),
              xadd(xadd(xmul(m[2], v.x), xmul(m[5], v.y)), xmul(m[8], v.z)));
}

__global__ void k_bake_instances(const BakeRecord* __restrict__ recs, u32 nrec, u32 total, float4* __restrict__ tri) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    u32 lo = 0, hi = nrec;   // the record whose thread range [first, first + e - b) holds t
    while (hi - lo > 1) { const u32 m = (lo + hi) / 2; if (recs[m].first <= t) lo = m; else hi = m; }
    const BakeRecord& r = recs[lo];
    const u32 i = t - r.first;
    const float* s = (const float*)r.tris + 36 * (size_t)i;   // st_mesh_triangle: positions[3][3], normals[3][3], uvs[3][2], tangents[3][4]
    float4* o = tri + 9 * ((size_t)r.b + i);
    for (int k = 0; k < 3; k++) {
        float3 p = aff_mat3(r.xf, f3(s[3 * k], s[3 * k + 1], s[3 * k + 2]));
        p = f3(xadd(p.x, r.xf[9]), xadd(p.y, r.xf[10]), xadd(p.z, r.xf[11]));
        const float3 n = xnorm(aff_mat3(r.nt, f3(s[9 + 3 * k], s[9 + 3 * k + 1], s[9 + 3 * k + 2])));
        const float3 tg = xnorm(aff_mat3(r.xf, f3(s[24 + 4 * k], s[24 + 4 * k + 1], s[24 + 4 * k + 2])));
        o[3 * k] = make_float4(p.x, p.y, p.z, s[18 + 2 * k]);
        o[3 * k + 1] = make_float4(n.x, n.y, n.z, s[18 + 2 * k + 1]);
        o[3 * k + 2] = make_float4(tg.x, tg.y, tg.z, xmul(s[24 + 4 * k + 3], r.sign));
    }
}

// The box of a child slot: lo in .xyz of bvh[slot], hi in .xyz of bvh[slot + 1]; the .w words (right_ptr, zero) are never written.
ST_DEV void store_slot(float4* bvh, u32 slot, float3 lo, float3 hi) {
    float* a = (float*)(bvh + slot); float* b = (float*)(bvh + slot + 1);
    a[0] = lo.x; a[1] = lo.y; a[2] = lo.z; b[0] = hi.x; b[1] = hi.y; b[2] = hi.z;
}

// one thread per leaf run {parent slot, first entry, entry count}: the box of its triangles' three positions
__global__ void k_refit_leaves(const uint4* __restrict__ runs, u32 n, const float4* __restrict__ tri, float4* bvh) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint4 r = runs[t];
    float3 lo = f3(kF32Max, kF32Max, kF32Max), hi = f3(-kF32Max, -kF32Max, -kF32Max);
    for (u32 i = 0; i < r.z; i++) {
        const u32 id = fbits(bvh[r.y + i].y);
        for (int k = 0; k < 3; k++) {
            const float4 p = tri[9 * (size_t)id + 3 * k];
            lo = f3(bmin(lo.x, p.x), bmin(lo.y, p.y), bmin(lo.z, p.z));
            hi = f3(bmax(hi.x, p.x), bmax(hi.y, p.y), bmax(hi.z, p.z));
        }
    }
    store_slot(bvh, r.x, lo, hi);
}

// one thread per internal node {ptr, parent slot} of one level: the union of its two child boxes goes into its parent's slot
__global__ void k_refit_nodes(const uint2* __restrict__ nodes, u32 n, float4* bvh) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint2 nd = nodes[t];
    const float4 a = bvh[nd.x], b = bvh[nd.x + 1], c = bvh[nd.x + 2], d = bvh[nd.x + 3];
    store_slot(bvh, nd.y, f3(bmin(a.x, c.x), bmin(a.y, c.y), bmin(a.z, c.z)), f3(bmax(b.x, d.x), bmax(b.y, d.y), bmax(b.z, d.z)));
}

void launch_bake_instances(const BakeRecord* recs, u32 nrec, u32 total, float4* triangles, cudaStream_t st) {
    if (!nrec || !total) return;
    k_bake_instances<<<(total + 127) / 128, 128, 0, st>>>(recs, nrec, total, triangles);
}

void launch_refit(const uint4* runs, u32 nruns, const uint2* nodes, const u32* level_begin, int levels, const float4* triangles, float4* bvh, cudaStream_t st) {
    if (nruns) k_refit_leaves<<<(nruns + 127) / 128, 128, 0, st>>>(runs, nruns, triangles, bvh);
    for (int l = 0; l < levels; l++) {   // deepest level first
        const u32 b = level_begin[l], n = level_begin[l + 1] - b;
        if (n) k_refit_nodes<<<(n + 127) / 128, 128, 0, st>>>(nodes + b, n, bvh);
    }
}

}  // namespace st
