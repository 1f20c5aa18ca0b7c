// raycast.cu -- closest-hit ray casting of a triangle mesh: a linear BVH (Karras 2012) built in three deterministic passes
// (Morton codes of the face centroids; per internal node its range, split and links; bottom-up boxes with one arrival
// counter per node), ordered stack traversal with a conservative slab test, the watertight ray/triangle test of Woop,
// Benthin & Wald (JCGT 2013), and a separate shading pass that turns hit records into the eval renders' outputs.  The caller
// (ops.mesh_bvh) sorts the codes in between.  Every fp32 operation of the codes, the boxes and the triangle test is an
// explicit round-to-nearest intrinsic, so the device build and the host build of tests/mesh_render_harness.py
// (-DPERF_HOST_HARNESS, where each entry point runs its body over host arrays in a serial loop) agree bit for bit.
// Rules and node layout: perfb200.h (perf_bvh_*, perf_mesh_*); restated in numpy in tests/mesh_render_oracle.py.
#include "common.cuh"

#ifdef __CUDA_ARCH__
#define PERF_DSUB_RN(a, b) __dsub_rn((a), (b))
#define PERF_DMUL_RN(a, b) __dmul_rn((a), (b))
#define PERF_FSQRT_RN(a) __fsqrt_rn(a)
#else
#define PERF_DSUB_RN(a, b) ((a) - (b))
#define PERF_DMUL_RN(a, b) ((a) * (b))
#define PERF_FSQRT_RN(a) sqrtf(a)
#endif

namespace perf {

// Traversal stack.  delta(i, j) of the extended key (code << 32 | index) is the length of the common prefix of a node's range
// and grows by at least 1 from an internal node to an internal child; it lies in [0, 64 + 31], so a root-to-leaf path has at
// most 96 internal nodes and the ordered traversal, which defers at most one sibling per level, never holds more than 96.
constexpr int BVH_STACK = 96;
static_assert(BVH_STACK >= 64 + 32, "the stack must hold one deferred sibling per level of a Karras tree");

// Slab-test slack: a box's [t_near, t_far] is widened by 2^-16 of its largest coordinate distance from the origin (over the
// largest direction component) and by 2^-16 of |t| itself before it is compared (see perfb200.h).
constexpr float BVH_SLACK = 1.52587890625e-05f;

struct BvhArgs {
    const float* pos; int64_t V;                    // [V,3]
    const int32_t* faces; int64_t F;                // [F,3]
    float lo[3], ext[3];                            // code box
    int64_t* codes;                                 // [F] Morton codes (perf_bvh_codes), sorted (perf_bvh_topology)
    int32_t* nodes;                                 // [F - 1, 16] (float box words + int32 links)
    int32_t* leaf_parent;                           // [F]
    const int32_t* order;                           // [F] face at each leaf position
    float* tris;                                    // [F, 12]
    int32_t* counters;                              // [F - 1], zero before perf_bvh_boxes
};

// ---------------------------------------------------------------- codes
__host__ __device__ __forceinline__ uint64_t bvh_spread(uint32_t v)
{
    uint64_t x = v & 0x1FFFFFull;
    x = (x | (x << 32)) & 0x1F00000000FFFFull;
    x = (x | (x << 16)) & 0x1F0000FF0000FFull;
    x = (x | (x << 8)) & 0x100F00F00F00F00Full;
    x = (x | (x << 4)) & 0x10C30C30C30C30C3ull;
    x = (x | (x << 2)) & 0x1249249249249249ull;
    return x;
}

// centroid c = ((p0 + p1) + p2) / 3; per axis u = (c - lo) / ext, q = min(2^21 - 1, floor(max(u, 0) * 2^21)), 0 when ext = 0;
// code = x in bits 3k, y in 3k + 1, z in 3k + 2.
__host__ __device__ __forceinline__ void bvh_code(const BvhArgs& a, int64_t f)
{
    uint32_t q[3];
    const int32_t i0 = a.faces[3 * f], i1 = a.faces[3 * f + 1], i2 = a.faces[3 * f + 2];
    for (int d = 0; d < 3; ++d) {
        const float c = PERF_FDIV_RN(PERF_FADD_RN(PERF_FADD_RN(a.pos[3 * (int64_t)i0 + d], a.pos[3 * (int64_t)i1 + d]),
                                                  a.pos[3 * (int64_t)i2 + d]), 3.0f);
        q[d] = 0;
        if (a.ext[d] > 0.0f) {
            float u = PERF_FMUL_RN(PERF_FDIV_RN(PERF_FSUB_RN(c, a.lo[d]), a.ext[d]), 2097152.0f);
            u = u > 0.0f ? u : 0.0f;
            q[d] = u >= 2097151.0f ? 2097151u : (uint32_t)u;
        }
    }
    a.codes[f] = (int64_t)(bvh_spread(q[0]) | (bvh_spread(q[1]) << 1) | (bvh_spread(q[2]) << 2));
}

// ---------------------------------------------------------------- topology
__host__ __device__ __forceinline__ int bvh_clz64(uint64_t x)
{
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return x ? __builtin_clzll(x) : 64;
#endif
}
__host__ __device__ __forceinline__ int bvh_clz32(uint32_t x)
{
#ifdef __CUDA_ARCH__
    return __clz((int)x);
#else
    return x ? __builtin_clz(x) : 32;
#endif
}

// delta(i, j): -1 outside [0, F), clz(code_i ^ code_j), or 64 + clz(i ^ j) for equal codes.
__host__ __device__ __forceinline__ int bvh_delta(const BvhArgs& a, int64_t i, int64_t j)
{
    if (j < 0 || j >= a.F) return -1;
    const uint64_t x = (uint64_t)a.codes[i] ^ (uint64_t)a.codes[j];
    return x ? bvh_clz64(x) : 64 + bvh_clz32((uint32_t)i ^ (uint32_t)j);
}

// Internal node i of F - 1 (Karras 2012, figure 4).  Child link c >= 0: internal node c; c < 0: leaf ~c.
__host__ __device__ __forceinline__ void bvh_node(const BvhArgs& a, int64_t i)
{
    const int d = bvh_delta(a, i, i + 1) > bvh_delta(a, i, i - 1) ? 1 : -1;
    const int dmin = bvh_delta(a, i, i - d);
    int64_t lmax = 2;
    while (bvh_delta(a, i, i + lmax * d) > dmin) lmax *= 2;
    int64_t l = 0;
    for (int64_t t = lmax / 2; t >= 1; t /= 2)
        if (bvh_delta(a, i, i + (l + t) * d) > dmin) l += t;
    const int64_t j = i + l * d;
    const int dnode = bvh_delta(a, i, j);
    int64_t s = 0;
    for (int64_t div = 2;; div *= 2) {
        const int64_t t = (l + div - 1) / div;
        if (bvh_delta(a, i, i + (s + t) * d) > dnode) s += t;
        if (t <= 1) break;
    }
    const int64_t g = i + s * d + (d < 0 ? -1 : 0);
    const int64_t lo = i < j ? i : j, hi = i < j ? j : i;
    int32_t* n = a.nodes + 16 * i;
    n[12] = lo == g ? ~(int32_t)g : (int32_t)g;
    n[13] = hi == g + 1 ? ~(int32_t)(g + 1) : (int32_t)(g + 1);
    if (lo == g) a.leaf_parent[g] = (int32_t)i; else a.nodes[16 * g + 14] = (int32_t)i;
    if (hi == g + 1) a.leaf_parent[g + 1] = (int32_t)i; else a.nodes[16 * (g + 1) + 14] = (int32_t)i;
    if (i == 0) n[14] = -1;
    n[15] = 0;
}

// ---------------------------------------------------------------- boxes
__host__ __device__ __forceinline__ float bvh_f(int32_t v) { float f; memcpy(&f, &v, 4); return f; }
__host__ __device__ __forceinline__ int32_t bvh_i(float v) { int32_t i; memcpy(&i, &v, 4); return i; }

__host__ __device__ __forceinline__ int bvh_arrive(int32_t* c)
{
#ifdef __CUDA_ARCH__
    __threadfence();
    const int old = atomicAdd((int*)c, 1);
    __threadfence();
    return old;
#else
    return (*c)++;
#endif
}
__host__ __device__ __forceinline__ int32_t bvh_load(const int32_t* p)
{
#ifdef __CUDA_ARCH__
    return __ldcg(p);                                   // the sibling's slot, written by another thread: bypass L1
#else
    return *p;
#endif
}

// Leaf at position i: triangle record, box; then up the tree, every node's box = min/max of its two child slots, computed by
// the second of the two threads to arrive.
__host__ __device__ __forceinline__ void bvh_leaf(const BvhArgs& a, int64_t i)
{
    const int32_t f = a.order[i];
    float box[6], p[3][3];
    for (int k = 0; k < 3; ++k)
        for (int d = 0; d < 3; ++d) p[k][d] = a.pos[3 * (int64_t)a.faces[3 * (int64_t)f + k] + d];
    float* t = a.tris + 12 * i;
    for (int k = 0; k < 3; ++k) {
        for (int d = 0; d < 3; ++d) t[4 * k + d] = p[k][d];
        t[4 * k + 3] = k == 0 ? bvh_f(f) : 0.0f;
    }
    for (int d = 0; d < 3; ++d) {
        box[d] = fminf(fminf(p[0][d], p[1][d]), p[2][d]);
        box[3 + d] = fmaxf(fmaxf(p[0][d], p[1][d]), p[2][d]);
    }
    if (a.F == 1) return;
    int32_t child = ~(int32_t)i, node = a.leaf_parent[i];
    while (node >= 0) {
        int32_t* n = a.nodes + 16 * (int64_t)node;
        const int side = n[12] == child ? 0 : 1;
        for (int d = 0; d < 6; ++d) n[6 * side + d] = bvh_i(box[d]);
        if (bvh_arrive(a.counters + node) == 0) return;
        const int32_t* o = n + 6 * (1 - side);
        for (int d = 0; d < 3; ++d) {
            box[d] = fminf(box[d], bvh_f(bvh_load(o + d)));
            box[3 + d] = fmaxf(box[3 + d], bvh_f(bvh_load(o + 3 + d)));
        }
        child = node;
        node = n[14];
    }
}

// ---------------------------------------------------------------- cast
struct Ray {
    float o[3], d[3], inv[3];                       // inv = 0 where the direction component is parallel (|d| < 2^-100)
    int kx, ky, kz;
    float sx, sy, sz, inv_dmax;
    float tmin;
};

__host__ __device__ __forceinline__ void ray_setup(Ray& r, float tmin)
{
    r.tmin = tmin;
    float ad[3];
    for (int d = 0; d < 3; ++d) {
        ad[d] = fabsf(r.d[d]);
        r.inv[d] = ad[d] >= 7.88860905e-31f ? PERF_FDIV_RN(1.0f, r.d[d]) : 0.0f;
    }
    r.kz = ad[0] >= ad[1] ? (ad[0] >= ad[2] ? 0 : 2) : (ad[1] >= ad[2] ? 1 : 2);
    r.kx = r.kz == 2 ? 0 : r.kz + 1;
    r.ky = r.kx == 2 ? 0 : r.kx + 1;
    if (r.d[r.kz] < 0.0f) { const int s = r.kx; r.kx = r.ky; r.ky = s; }
    r.sx = PERF_FDIV_RN(r.d[r.kx], r.d[r.kz]);
    r.sy = PERF_FDIV_RN(r.d[r.ky], r.d[r.kz]);
    r.sz = PERF_FDIV_RN(1.0f, r.d[r.kz]);
    r.inv_dmax = ad[r.kz] > 0.0f ? PERF_FDIV_RN(1.0f, ad[r.kz]) : 0.0f;
}

// Woop, Benthin & Wald, two-sided: true with (t, b1, b2) when the ray hits the triangle with t in [tmin, tmax].
__host__ __device__ __forceinline__ float ray_pick(const float (&v)[3], int k) { return k == 0 ? v[0] : (k == 1 ? v[1] : v[2]); }

__host__ __device__ __forceinline__ bool ray_triangle(const Ray& r, const float* tri, float tmax, float& t, float& b1, float& b2)
{
    float A[3], B[3], C[3];
    for (int d = 0; d < 3; ++d) {
        A[d] = PERF_FSUB_RN(tri[d], r.o[d]);
        B[d] = PERF_FSUB_RN(tri[4 + d], r.o[d]);
        C[d] = PERF_FSUB_RN(tri[8 + d], r.o[d]);
    }
    const float ax = PERF_FSUB_RN(ray_pick(A, r.kx), PERF_FMUL_RN(r.sx, ray_pick(A, r.kz))), ay = PERF_FSUB_RN(ray_pick(A, r.ky), PERF_FMUL_RN(r.sy, ray_pick(A, r.kz)));
    const float bx = PERF_FSUB_RN(ray_pick(B, r.kx), PERF_FMUL_RN(r.sx, ray_pick(B, r.kz))), by = PERF_FSUB_RN(ray_pick(B, r.ky), PERF_FMUL_RN(r.sy, ray_pick(B, r.kz)));
    const float cx = PERF_FSUB_RN(ray_pick(C, r.kx), PERF_FMUL_RN(r.sx, ray_pick(C, r.kz))), cy = PERF_FSUB_RN(ray_pick(C, r.ky), PERF_FMUL_RN(r.sy, ray_pick(C, r.kz)));
    float U = PERF_FSUB_RN(PERF_FMUL_RN(cx, by), PERF_FMUL_RN(cy, bx));
    float V = PERF_FSUB_RN(PERF_FMUL_RN(ax, cy), PERF_FMUL_RN(ay, cx));
    float W = PERF_FSUB_RN(PERF_FMUL_RN(bx, ay), PERF_FMUL_RN(by, ax));
    if (U == 0.0f || V == 0.0f || W == 0.0f) {          // on an edge in fp32: decide it in fp64 (products of fp32 are exact)
        U = (float)PERF_DSUB_RN(PERF_DMUL_RN((double)cx, (double)by), PERF_DMUL_RN((double)cy, (double)bx));
        V = (float)PERF_DSUB_RN(PERF_DMUL_RN((double)ax, (double)cy), PERF_DMUL_RN((double)ay, (double)cx));
        W = (float)PERF_DSUB_RN(PERF_DMUL_RN((double)bx, (double)ay), PERF_DMUL_RN((double)by, (double)ax));
    }
    if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return false;
    const float det = PERF_FADD_RN(PERF_FADD_RN(U, V), W);
    if (det == 0.0f) return false;
    const float az = PERF_FMUL_RN(r.sz, ray_pick(A, r.kz)), bz = PERF_FMUL_RN(r.sz, ray_pick(B, r.kz)), cz = PERF_FMUL_RN(r.sz, ray_pick(C, r.kz));
    const float T = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(U, az), PERF_FMUL_RN(V, bz)), PERF_FMUL_RN(W, cz));
    t = PERF_FDIV_RN(T, det);
    if (!(t >= r.tmin && t <= tmax)) return false;
    b1 = PERF_FDIV_RN(V, det);
    b2 = PERF_FDIV_RN(W, det);
    return true;
}

// Conservative slab test of box (lo xyz, hi xyz) against [tmin, tbest]: false when the box is culled, else true with the
// widened entry distance tn.  A parallel axis (inv = 0) culls when the origin lies outside its slab by more than the slack.
__host__ __device__ __forceinline__ bool ray_box(const Ray& r, const float* b, float tbest, float& tn)
{
    float dl[3], dh[3], m = 0.0f, tf = INFINITY;
    tn = -INFINITY;
    for (int d = 0; d < 3; ++d) {
        dl[d] = b[d] - r.o[d]; dh[d] = b[3 + d] - r.o[d];
        m = fmaxf(m, fmaxf(fabsf(dl[d]), fabsf(dh[d])));
    }
    const float mw = m * BVH_SLACK, slack = mw * r.inv_dmax;
    for (int d = 0; d < 3; ++d) {
        if (r.inv[d] == 0.0f) {
            if (dl[d] > mw || dh[d] < -mw) return false;
        } else {
            const float t0 = dl[d] * r.inv[d], t1 = dh[d] * r.inv[d];
            tn = fmaxf(tn, fminf(t0, t1));
            tf = fminf(tf, fmaxf(t0, t1));
        }
    }
    tn = tn - slack - fabsf(tn) * BVH_SLACK;
    tf = tf + slack + fabsf(tf) * BVH_SLACK;
    return !(tn > tf || tn > tbest || tf < r.tmin);
}

// Closest hit of one ray: record (t, face, b1, b2), face -1 and t = +inf on a miss; minimises (t, face) lexicographically.
__host__ __device__ __forceinline__ void ray_cast(const int32_t* __restrict__ nodes, const float* __restrict__ tris, int64_t F,
                                                  const Ray& r, float tmax, float4* rec)
{
    float bt = tmax, bb1 = 0.0f, bb2 = 0.0f;
    int32_t bf = -1;
    auto leaf = [&](int32_t l) {
        const float* tri = tris + 12 * (int64_t)l;
        float t, b1, b2;
        if (ray_triangle(r, tri, bt, t, b1, b2)) {
            const int32_t f = bvh_i(tri[3]);
            if (bf < 0 || t < bt || f < bf) { bt = t; bf = f; bb1 = b1; bb2 = b2; }
        }
    };
    if (F == 1) leaf(0);
    if (F >= 2) {
        int32_t stack_node[BVH_STACK];
        float stack_t[BVH_STACK];
        int sp = 0;
        int32_t node = 0;
        for (;;) {
            const int32_t* n = nodes + 16 * (int64_t)node;
            float box[12];
            for (int k = 0; k < 12; ++k) box[k] = bvh_f(n[k]);
            const int32_t c0 = n[12], c1 = n[13];
            float t0, t1;
            const bool h0 = ray_box(r, box, bt, t0), h1 = ray_box(r, box + 6, bt, t1);
            int32_t next = INT32_MIN;
            if (h0 && h1) {
                const bool first0 = t0 <= t1;
                const int32_t cn = first0 ? c0 : c1, cf = first0 ? c1 : c0;
                const float tf = first0 ? t1 : t0;
                if (cf < 0) leaf(~cf); else { stack_node[sp] = cf; stack_t[sp] = tf; ++sp; }
                if (cn < 0) leaf(~cn); else next = cn;
            } else if (h0) {
                if (c0 < 0) leaf(~c0); else next = c0;
            } else if (h1) {
                if (c1 < 0) leaf(~c1); else next = c1;
            }
            if (next == INT32_MIN) {
                while (sp > 0) {
                    --sp;
                    if (stack_t[sp] <= bt) { next = stack_node[sp]; break; }
                }
                if (next == INT32_MIN) break;
            }
            node = next;
        }
    }
    *rec = make_float4(bf < 0 ? INFINITY : bt, bvh_f(bf), bf < 0 ? 0.0f : bb1, bf < 0 ? 0.0f : bb2);
}

struct CastArgs {
    const int32_t* nodes; const float* tris; int64_t F;
    const float* o; const float* d; int64_t R;
    float tmin, tmax;
    float pose[12]; int H, W, row0, rows;           // pano: rotation rows and translation (perf_raygen_pano's Pose)
    float4* hits;
};

__host__ __device__ __forceinline__ void cast_ray(const CastArgs& a, int64_t i)
{
    Ray r;
    for (int d = 0; d < 3; ++d) { r.o[d] = a.o[3 * i + d]; r.d[d] = a.d[3 * i + d]; }
    ray_setup(r, a.tmin);
    ray_cast(a.nodes, a.tris, a.F, r, a.tmax, a.hits + i);
}

// Pixel (row0 + y, x) of the pano window: the ray perf_raygen_pano generates there (common.cuh pano_dir + rotate).
__host__ __device__ __forceinline__ void cast_pixel(const CastArgs& a, int y, int x)
{
    Ray r;
    float cx, cy, cz;
    pano_dir(a.row0 + y, x, a.H, a.W, cx, cy, cz);
    const float rot[9] = {a.pose[0], a.pose[1], a.pose[2], a.pose[3], a.pose[4], a.pose[5], a.pose[6], a.pose[7], a.pose[8]};
    rotate(rot, cx, cy, cz, r.d[0], r.d[1], r.d[2]);
    r.o[0] = a.pose[9]; r.o[1] = a.pose[10]; r.o[2] = a.pose[11];
    ray_setup(r, a.tmin);
    ray_cast(a.nodes, a.tris, a.F, r, a.tmax, a.hits + (int64_t)y * a.W + x);
}

// ---------------------------------------------------------------- shade
struct ShadeArgs {
    const float4* hits; int64_t R;
    const float* d;                                 // [R,3] ray directions (back-face test)
    const float* pos; int64_t V;
    const int32_t* faces; int64_t F;
    const uint8_t* colors;                          // [V,3] nullable
    const float* normals;                           // [V,3] nullable
    const float* uv;                                // [F,3,2] nullable (with texture)
    const uint8_t* texture; int T;                  // [T,T,3]
    float* rgb; float* dist; float* op; float* nrm; uint8_t* back;
    const uint8_t* ntex;                            // [T,T,3] normal texture (shade_ray<true> only)
};

__host__ __device__ __forceinline__ float shade_texel(const ShadeArgs& a, int x, int y, int c)
{
    x = x < 0 ? 0 : (x >= a.T ? a.T - 1 : x);
    y = y < 0 ? 0 : (y >= a.T ? a.T - 1 : y);
    return (float)a.texture[3 * ((int64_t)y * a.T + x) + c];
}
// The same addressing in the normal texture.
__host__ __device__ __forceinline__ float shade_ntexel(const ShadeArgs& a, int x, int y, int c)
{
    x = x < 0 ? 0 : (x >= a.T ? a.T - 1 : x);
    y = y < 0 ? 0 : (y >= a.T ? a.T - 1 : y);
    return (float)a.ntex[3 * ((int64_t)y * a.T + x) + c];
}

// The shading normal of a hit at barycentrics w on the face of vertices v and geometric normal g = (p1 - p0) x (p2 - p0):
// the blend of the vertex normals, or g without them, normalised (0 when the blend is 0).  The mesh shade and the normal
// texture bake (the normal of the full-resolution surface it encodes) share it.
__host__ __device__ __forceinline__ void shade_normal(const float* normals, const int32_t (&v)[3], const float (&g)[3],
                                                      const float (&w)[3], float (&n)[3])
{
    for (int d = 0; d < 3; ++d) {
        n[d] = g[d];
        if (normals)
            n[d] = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], normals[3 * (int64_t)v[0] + d]),
                                             PERF_FMUL_RN(w[1], normals[3 * (int64_t)v[1] + d])),
                                PERF_FMUL_RN(w[2], normals[3 * (int64_t)v[2] + d]));
    }
    const float nn = PERF_FSQRT_RN(PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(n[0], n[0]), PERF_FMUL_RN(n[1], n[1])), PERF_FMUL_RN(n[2], n[2])));
    for (int d = 0; d < 3; ++d) n[d] = nn > 0.0f ? PERF_FDIV_RN(n[d], nn) : 0.0f;
}

// ---------------------------------------------------------------- normal texture (perfb200.h, perf_normal_texture_bake)
__host__ __device__ __forceinline__ float nt_dot(const float (&a)[3], const float (&b)[3])
{
    return PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(a[0], b[0]), PERF_FMUL_RN(a[1], b[1])), PERF_FMUL_RN(a[2], b[2]));
}
__host__ __device__ __forceinline__ void nt_cross(const float (&a)[3], const float (&b)[3], float (&c)[3])
{
    c[0] = PERF_FSUB_RN(PERF_FMUL_RN(a[1], b[2]), PERF_FMUL_RN(a[2], b[1]));
    c[1] = PERF_FSUB_RN(PERF_FMUL_RN(a[2], b[0]), PERF_FMUL_RN(a[0], b[2]));
    c[2] = PERF_FSUB_RN(PERF_FMUL_RN(a[0], b[1]), PERF_FMUL_RN(a[1], b[0]));
}

// MikkTSpace's corner frames for per-face charts (no corner is welded across faces) of a face with edges e1, e2, geometric
// normal g = e1 x e2 and corner uv[6]: the face tangent T_f from the uv differences, per corner n_k (the vertex normal, or
// the unit geometric normal without vertex normals) and t_k = T_f made orthogonal to n_k and normalised.
__host__ __device__ __forceinline__ void nt_corners(const float (&e1)[3], const float (&e2)[3], const float (&g)[3], const float* normals,
                                                    const int32_t (&v)[3], const float* uv, float (&nk)[3][3], float (&tk)[3][3])
{
    const float du1 = PERF_FSUB_RN(uv[2], uv[0]), dv1 = PERF_FSUB_RN(uv[3], uv[1]);
    const float du2 = PERF_FSUB_RN(uv[4], uv[0]), dv2 = PERF_FSUB_RN(uv[5], uv[1]);
    const float den = PERF_FSUB_RN(PERF_FMUL_RN(du1, dv2), PERF_FMUL_RN(du2, dv1));
    float tf[3], gh[3];
    for (int d = 0; d < 3; ++d) tf[d] = PERF_FDIV_RN(PERF_FSUB_RN(PERF_FMUL_RN(dv2, e1[d]), PERF_FMUL_RN(dv1, e2[d])), den);
    const float gl = PERF_FSQRT_RN(nt_dot(g, g));
    for (int d = 0; d < 3; ++d) gh[d] = gl > 0.0f ? PERF_FDIV_RN(g[d], gl) : 0.0f;
    for (int k = 0; k < 3; ++k) {
        float u[3];
        for (int d = 0; d < 3; ++d) nk[k][d] = normals ? normals[3 * (int64_t)v[k] + d] : gh[d];
        const float s = nt_dot(nk[k], tf);
        for (int d = 0; d < 3; ++d) u[d] = PERF_FSUB_RN(tf[d], PERF_FMUL_RN(nk[k][d], s));
        const float ul = PERF_FSQRT_RN(nt_dot(u, u));
        for (int d = 0; d < 3; ++d) tk[k][d] = ul > 0.0f ? PERF_FDIV_RN(u[d], ul) : 0.0f;
    }
}

// The frame at barycentrics w: the unnormalised blends n = sum w_k n_k, t = sum w_k t_k of nt_corners and the bitangent
// b = n x t (sign +1: every chart has positive area).
__host__ __device__ __forceinline__ void nt_frame(const float (&e1)[3], const float (&e2)[3], const float (&g)[3], const float* normals,
                                                  const int32_t (&v)[3], const float* uv, const float (&w)[3], float (&t)[3],
                                                  float (&b)[3], float (&n)[3])
{
    float nk[3][3], tk[3][3];
    nt_corners(e1, e2, g, normals, v, uv, nk, tk);
    for (int d = 0; d < 3; ++d) {
        n[d] = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], nk[0][d]), PERF_FMUL_RN(w[1], nk[1][d])), PERF_FMUL_RN(w[2], nk[2][d]));
        t[d] = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], tk[0][d]), PERF_FMUL_RN(w[1], tk[1][d])), PERF_FMUL_RN(w[2], tk[2][d]));
    }
    nt_cross(n, t, b);
}

// Encodes the unit normal N in the frame (t, b, n): c = [t b n]^-1 N by Cramer's rule, normalised, stored as
// floor((c + 1) 127.5 + 0.5) clamped to [0, 255].  False (the caller keeps the flat texel) for a degenerate frame,
// |det| <= 1e-12 |t| |b| |n|, or c = 0.
__host__ __device__ __forceinline__ bool nt_encode(const float (&t)[3], const float (&b)[3], const float (&n)[3], const float (&N)[3],
                                                   uint8_t* out)
{
    float bn[3], Nn[3], bN[3];
    nt_cross(b, n, bn);
    const float det = nt_dot(t, bn);
    const float lim = PERF_FMUL_RN(PERF_FMUL_RN(PERF_FMUL_RN(1e-12f, PERF_FSQRT_RN(nt_dot(t, t))), PERF_FSQRT_RN(nt_dot(b, b))),
                                   PERF_FSQRT_RN(nt_dot(n, n)));
    if (!(fabsf(det) > lim)) return false;
    nt_cross(N, n, Nn);
    nt_cross(b, N, bN);
    const float c[3] = {PERF_FDIV_RN(nt_dot(N, bn), det), PERF_FDIV_RN(nt_dot(t, Nn), det), PERF_FDIV_RN(nt_dot(t, bN), det)};
    const float cl = PERF_FSQRT_RN(nt_dot(c, c));
    if (!(cl > 0.0f)) return false;
    for (int k = 0; k < 3; ++k) {
        const float q = floorf(PERF_FADD_RN(PERF_FMUL_RN(PERF_FADD_RN(PERF_FDIV_RN(c[k], cl), 1.0f), 127.5f), 0.5f));
        out[k] = (uint8_t)(q < 0.0f ? 0.0f : (q > 255.0f ? 255.0f : q));
    }
    return true;
}

// The normal texture applied to a hit (the shading normal n of shade_normal on input): a bilinear lookup of the bytes at
// the blended uv with the albedo's addressing, c = texel / 127.5 - 1, n = normalise((c.x t + c.y b) + c.z n_frame); n is
// left as it is when that vector is 0 (a degenerate frame).
__host__ __device__ __forceinline__ void shade_normal_texture(const ShadeArgs& a, int32_t f, const float (&e1)[3], const float (&e2)[3],
                                                              const float (&g)[3], const int32_t (&v)[3], const float (&w)[3],
                                                              float (&n)[3])
{
    const float* uv = a.uv + 6 * (int64_t)f;
    const float u = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], uv[0]), PERF_FMUL_RN(w[1], uv[2])), PERF_FMUL_RN(w[2], uv[4]));
    const float vv = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], uv[1]), PERF_FMUL_RN(w[1], uv[3])), PERF_FMUL_RN(w[2], uv[5]));
    const float T = (float)a.T;
    const float x = PERF_FSUB_RN(PERF_FMUL_RN(u, T), 0.5f), y = PERF_FSUB_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, vv), T), 0.5f);
    const float x0 = floorf(x), y0 = floorf(y), fx = PERF_FSUB_RN(x, x0), fy = PERF_FSUB_RN(y, y0);
    const int ix = (int)x0, iy = (int)y0;
    float c[3], t[3], b[3], m[3], N[3];
    for (int k = 0; k < 3; ++k) {
        const float top = PERF_FADD_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, fx), shade_ntexel(a, ix, iy, k)),
                                       PERF_FMUL_RN(fx, shade_ntexel(a, ix + 1, iy, k)));
        const float bot = PERF_FADD_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, fx), shade_ntexel(a, ix, iy + 1, k)),
                                       PERF_FMUL_RN(fx, shade_ntexel(a, ix + 1, iy + 1, k)));
        c[k] = PERF_FSUB_RN(PERF_FDIV_RN(PERF_FADD_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, fy), top), PERF_FMUL_RN(fy, bot)), 127.5f), 1.0f);
    }
    nt_frame(e1, e2, g, a.normals, v, uv, w, t, b, m);
    for (int d = 0; d < 3; ++d)
        N[d] = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(c[0], t[d]), PERF_FMUL_RN(c[1], b[d])), PERF_FMUL_RN(c[2], m[d]));
    const float nl = PERF_FSQRT_RN(nt_dot(N, N));
    if (nl > 0.0f)
        for (int d = 0; d < 3; ++d) n[d] = PERF_FDIV_RN(N[d], nl);
}

template <bool NT>
__host__ __device__ __forceinline__ void shade_ray(const ShadeArgs& a, int64_t i)
{
    const float4 h = a.hits[i];
    const int32_t f = bvh_i(h.y);
    float rgb[3] = {0.0f, 0.0f, 0.0f}, n[3] = {0.0f, 0.0f, 0.0f}, dist = 0.0f, op = 0.0f;
    uint8_t back = 0;
    if (f >= 0) {
        op = 1.0f;
        dist = h.x;
        const float b1 = h.z, b2 = h.w, b0 = PERF_FSUB_RN(PERF_FSUB_RN(1.0f, b1), b2);
        const float w[3] = {b0, b1, b2};
        int32_t v[3];
        float p[3][3];
        for (int k = 0; k < 3; ++k) {
            v[k] = a.faces[3 * (int64_t)f + k];
            for (int d = 0; d < 3; ++d) p[k][d] = a.pos[3 * (int64_t)v[k] + d];
        }
        float e1[3], e2[3];
        for (int d = 0; d < 3; ++d) { e1[d] = PERF_FSUB_RN(p[1][d], p[0][d]); e2[d] = PERF_FSUB_RN(p[2][d], p[0][d]); }
        const float g[3] = {PERF_FSUB_RN(PERF_FMUL_RN(e1[1], e2[2]), PERF_FMUL_RN(e1[2], e2[1])),
                            PERF_FSUB_RN(PERF_FMUL_RN(e1[2], e2[0]), PERF_FMUL_RN(e1[0], e2[2])),
                            PERF_FSUB_RN(PERF_FMUL_RN(e1[0], e2[1]), PERF_FMUL_RN(e1[1], e2[0]))};
        const float* dir = a.d + 3 * i;
        const float dg = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(dir[0], g[0]), PERF_FMUL_RN(dir[1], g[1])), PERF_FMUL_RN(dir[2], g[2]));
        back = dg > 0.0f;
        shade_normal(a.normals, v, g, w, n);
        if (NT) shade_normal_texture(a, f, e1, e2, g, v, w, n);
        if (a.texture) {
            // texel (x, y) of row y (row 0 at v = 1) has its centre at u = (x + 0.5) / T, v = 1 - (y + 0.5) / T
            const float* uv = a.uv + 6 * (int64_t)f;
            const float u = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], uv[0]), PERF_FMUL_RN(w[1], uv[2])), PERF_FMUL_RN(w[2], uv[4]));
            const float vv = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], uv[1]), PERF_FMUL_RN(w[1], uv[3])), PERF_FMUL_RN(w[2], uv[5]));
            const float T = (float)a.T;
            const float x = PERF_FSUB_RN(PERF_FMUL_RN(u, T), 0.5f), y = PERF_FSUB_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, vv), T), 0.5f);
            const float x0 = floorf(x), y0 = floorf(y), fx = PERF_FSUB_RN(x, x0), fy = PERF_FSUB_RN(y, y0);
            const int ix = (int)x0, iy = (int)y0;
            for (int c = 0; c < 3; ++c) {
                const float top = PERF_FADD_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, fx), shade_texel(a, ix, iy, c)), PERF_FMUL_RN(fx, shade_texel(a, ix + 1, iy, c)));
                const float bot = PERF_FADD_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, fx), shade_texel(a, ix, iy + 1, c)), PERF_FMUL_RN(fx, shade_texel(a, ix + 1, iy + 1, c)));
                rgb[c] = PERF_FDIV_RN(PERF_FADD_RN(PERF_FMUL_RN(PERF_FSUB_RN(1.0f, fy), top), PERF_FMUL_RN(fy, bot)), 255.0f);
            }
        } else if (a.colors) {
            for (int c = 0; c < 3; ++c)
                rgb[c] = PERF_FDIV_RN(PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(w[0], (float)a.colors[3 * (int64_t)v[0] + c]),
                                                                PERF_FMUL_RN(w[1], (float)a.colors[3 * (int64_t)v[1] + c])),
                                                   PERF_FMUL_RN(w[2], (float)a.colors[3 * (int64_t)v[2] + c])), 255.0f);
        }
    }
    // the eval renders' background rule (perf_render_pano): distance += 5 (1 - opacity), rgb += 0.5 (1 - opacity)
    const float miss = PERF_FSUB_RN(1.0f, op);
    for (int c = 0; c < 3; ++c) {
        a.rgb[3 * i + c] = PERF_FADD_RN(rgb[c], PERF_FMUL_RN(0.5f, miss));
        a.nrm[3 * i + c] = n[c];
    }
    a.dist[i] = PERF_FADD_RN(dist, PERF_FMUL_RN(5.0f, miss));
    a.op[i] = op;
    a.back[i] = back;
}

// ---------------------------------------------------------------- normal texture bake
struct BakeArgs {
    const int32_t* nodes; const float* tris; int64_t hF;  // the high mesh's BVH
    const float* hpos; const int32_t* hfaces; const float* hnormals;  // the high mesh ([V,3] normals nullable)
    const float* pos; const int32_t* faces; const float* normals; const float* uv;  // the low mesh (normals nullable)
    const int32_t* face; const float* point; int64_t N;  // the texels (perf_atlas_texels)
    float dist;
    uint8_t* texel; float* offset;
};

__host__ __device__ __forceinline__ void load_face(const float* pos, const int32_t* faces, int32_t f, int32_t (&v)[3], float (&p)[3][3],
                                                   float (&e1)[3], float (&e2)[3], float (&g)[3])
{
    for (int k = 0; k < 3; ++k) {
        v[k] = faces[3 * (int64_t)f + k];
        for (int d = 0; d < 3; ++d) p[k][d] = pos[3 * (int64_t)v[k] + d];
    }
    for (int d = 0; d < 3; ++d) { e1[d] = PERF_FSUB_RN(p[1][d], p[0][d]); e2[d] = PERF_FSUB_RN(p[2][d], p[0][d]); }
    nt_cross(e1, e2, g);
}

// Texel i: barycentrics of its point on its low face, casts along +g and -g (unit geometric normal) over [0, dist] into the
// high mesh, the high mesh's shading normal at the nearer hit (+g on a tie), encoded in the low face's frame.
__host__ __device__ __forceinline__ void bake_texel(const BakeArgs& a, int64_t i)
{
    uint8_t out[3] = {128, 128, 255};
    float off = INFINITY;
    const int32_t f = a.face[i];
    int32_t v[3];
    float p[3][3], e1[3], e2[3], g[3];
    if (f >= 0) load_face(a.pos, a.faces, f, v, p, e1, e2, g);
    const float G = f >= 0 ? nt_dot(g, g) : 0.0f;
    if (G > 0.0f) {
        float q[3], qe2[3], e1q[3];
        for (int d = 0; d < 3; ++d) q[d] = PERF_FSUB_RN(a.point[3 * i + d], p[0][d]);
        nt_cross(q, e2, qe2);
        nt_cross(e1, q, e1q);
        const float b1 = PERF_FDIV_RN(nt_dot(qe2, g), G), b2 = PERF_FDIV_RN(nt_dot(e1q, g), G);
        const float w[3] = {PERF_FSUB_RN(PERF_FSUB_RN(1.0f, b1), b2), b1, b2};
        const float gl = PERF_FSQRT_RN(G);
        float gh[3];
        for (int d = 0; d < 3; ++d) gh[d] = PERF_FDIV_RN(g[d], gl);
        // one cast at a time: a single call site keeps one traversal stack in the frame
        float4 best = make_float4(INFINITY, bvh_f(-1), 0.0f, 0.0f);
        int side = 0;
#pragma unroll 1
        for (int s = 0; s < 2; ++s) {
            Ray r;
            for (int d = 0; d < 3; ++d) { r.o[d] = a.point[3 * i + d]; r.d[d] = s ? -gh[d] : gh[d]; }
            ray_setup(r, 0.0f);
            float4 rec;
            ray_cast(a.nodes, a.tris, a.hF, r, a.dist, &rec);
            if (bvh_i(rec.y) >= 0 && (bvh_i(best.y) < 0 || rec.x < best.x)) { best = rec; side = s; }
        }
        const int32_t hf = bvh_i(best.y);
        if (hf >= 0) {
            off = side ? -best.x : best.x;
            int32_t hv[3];
            float hp[3][3], he1[3], he2[3], hg[3], N[3], t[3], b[3], n[3];
            load_face(a.hpos, a.hfaces, hf, hv, hp, he1, he2, hg);
            const float hw[3] = {PERF_FSUB_RN(PERF_FSUB_RN(1.0f, best.z), best.w), best.z, best.w};
            shade_normal(a.hnormals, hv, hg, hw, N);
            nt_frame(e1, e2, g, a.normals, v, a.uv + 6 * (int64_t)f, w, t, b, n);
            uint8_t c[3];
            if (nt_encode(t, b, n, N, c))
                for (int k = 0; k < 3; ++k) out[k] = c[k];
        }
    }
    for (int k = 0; k < 3; ++k) a.texel[3 * i + k] = out[k];
    a.offset[i] = off;
}

// ---------------------------------------------------------------- corner tangents (perf_mesh_corner_tangents)
struct TangentArgs { const float* pos; const int32_t* faces; const float* normals; const float* uv; int64_t F; float* out; };

// Face f: the unit corner tangents t_k of nt_corners, the ones the normal texture is baked and shaded with.
__host__ __device__ __forceinline__ void corner_tangents(const TangentArgs& a, int64_t f)
{
    int32_t v[3];
    float p[3][3], e1[3], e2[3], g[3], nk[3][3], tk[3][3];
    load_face(a.pos, a.faces, (int32_t)f, v, p, e1, e2, g);
    nt_corners(e1, e2, g, a.normals, v, a.uv + 6 * f, nk, tk);
    for (int k = 0; k < 3; ++k)
        for (int d = 0; d < 3; ++d) a.out[9 * f + 3 * k + d] = tk[k][d];
}

// ---------------------------------------------------------------- kernels
enum { BVH_CODES, BVH_TOPOLOGY, BVH_BOXES };

template <int S>
__host__ __device__ __forceinline__ void bvh_body(const BvhArgs& a, int64_t i)
{
    if (S == BVH_CODES) bvh_code(a, i);
    else if (S == BVH_TOPOLOGY) bvh_node(a, i);
    else bvh_leaf(a, i);
}

template <int S>
__global__ void __launch_bounds__(128) bvh_kernel(const BvhArgs a, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) bvh_body<S>(a, i);
}

__global__ void __launch_bounds__(128) mesh_cast_kernel(const CastArgs a)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.R) cast_ray(a, i);
}

// Pano: a 128-thread block covers a 16 x 8 pixel tile, each warp an 8 x 4 patch of it, so that a warp's rays traverse
// the same nodes.
constexpr int PANO_TX = 16, PANO_TY = 8;
__global__ void __launch_bounds__(128) mesh_cast_pano_kernel(const CastArgs a)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int x = blockIdx.x * PANO_TX + (warp & 1) * 8 + (lane & 7);
    const int y = blockIdx.y * PANO_TY + (warp >> 1) * 4 + (lane >> 3);
    if (x < a.W && y < a.rows) cast_pixel(a, y, x);
}

__global__ void __launch_bounds__(128) mesh_shade_kernel(const ShadeArgs a)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.R) shade_ray<false>(a, i);
}

__global__ void __launch_bounds__(128) mesh_shade_normal_texture_kernel(const ShadeArgs a)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.R) shade_ray<true>(a, i);
}

// One thread per texel in the atlas's Morton order: a warp holds neighbouring texels of one or two faces, whose rays are
// parallel and start close together, so they traverse the same nodes.
__global__ void __launch_bounds__(128) normal_texture_bake_kernel(const BakeArgs a)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.N) bake_texel(a, i);
}

__global__ void __launch_bounds__(128) mesh_corner_tangents_kernel(const TangentArgs a)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f < a.F) corner_tangents(a, f);
}

// The product library launches the kernels; the test harness build runs the same bodies over host arrays.
template <int S>
static int bvh_run(const BvhArgs& a, int64_t n, void* stream)
{
    if (n <= 0) return PERF_OK;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < n; ++i) bvh_body<S>(a, i);
#else
    bvh_kernel<S><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, n);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

}  // namespace perf

using namespace perf;

static int bvh_fill(BvhArgs& a, const float* vertices, uint64_t V, const int32_t* faces, uint64_t F)
{
    PERF_CHECK_ARG(V < (1ull << 31) && F < (1ull << 30), "mesh of %llu vertices / %llu faces: needs V < 2^31 and F < 2^30",
                   (unsigned long long)V, (unsigned long long)F);
    PERF_CHECK_ARG(F == 0 || (vertices && faces), "NULL vertices or faces");
    memset(&a, 0, sizeof(a));
    a.pos = vertices; a.V = (int64_t)V; a.faces = faces; a.F = (int64_t)F;
    return PERF_OK;
}

static int cast_fill(CastArgs& a, const int32_t* nodes, const float* tris, uint64_t F, float t_min, float t_max, void* hits)
{
    PERF_CHECK_ARG(F < (1ull << 30), "BVH of %llu faces: needs F < 2^30", (unsigned long long)F);
    PERF_CHECK_ARG(F == 0 || (tris && (F == 1 || nodes)), "NULL BVH arrays");
    PERF_CHECK_ARG(hits, "NULL hits");
    PERF_CHECK_ARG(!(t_min != t_min) && !(t_max != t_max), "NaN ray interval");
    memset(&a, 0, sizeof(a));
    a.nodes = nodes; a.tris = tris; a.F = (int64_t)F; a.tmin = t_min; a.tmax = t_max; a.hits = (float4*)hits;
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

int perf_bvh_codes(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const float* h_lo3, const float* h_hi3,
                   int64_t* d_codes, void* stream)
{
    BvhArgs a;
    int rc = bvh_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(F == 0 || (d_codes && h_lo3 && h_hi3), "NULL pointer");
    if (F) {
        for (int d = 0; d < 3; ++d) {
            PERF_CHECK_ARG(h_lo3[d] <= h_hi3[d], "code box: lo > hi on axis %d", d);
            a.lo[d] = h_lo3[d]; a.ext[d] = h_hi3[d] - h_lo3[d];
            PERF_CHECK_ARG(a.ext[d] < INFINITY, "code box: infinite extent on axis %d", d);
        }
    }
    a.codes = d_codes;
    return bvh_run<BVH_CODES>(a, (int64_t)F, stream);
}

int perf_bvh_topology(const int64_t* d_sorted_codes, uint64_t F, int32_t* d_nodes, int32_t* d_leaf_parent, void* stream)
{
    BvhArgs a;
    int rc = bvh_fill(a, nullptr, 0, nullptr, 0); if (rc) return rc;
    PERF_CHECK_ARG(F < (1ull << 30), "%llu faces: needs F < 2^30", (unsigned long long)F);
    PERF_CHECK_ARG(F < 2 || (d_sorted_codes && d_nodes && d_leaf_parent), "NULL pointer");
    a.F = (int64_t)F; a.codes = (int64_t*)d_sorted_codes; a.nodes = d_nodes; a.leaf_parent = d_leaf_parent;
    if (F == 1) {
        PERF_CHECK_ARG(d_leaf_parent, "NULL pointer");
#ifdef PERF_HOST_HARNESS
        d_leaf_parent[0] = -1;
#else
        PERF_CUDA(cudaMemsetAsync(d_leaf_parent, 0xFF, sizeof(int32_t), (cudaStream_t)stream));
#endif
        return PERF_OK;
    }
    return bvh_run<BVH_TOPOLOGY>(a, F < 2 ? 0 : (int64_t)F - 1, stream);
}

int perf_bvh_boxes(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_order,
                   const int32_t* d_leaf_parent, int32_t* d_nodes, float* d_tris, int32_t* d_counters, void* stream)
{
    BvhArgs a;
    int rc = bvh_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(F == 0 || (d_order && d_leaf_parent && d_tris && (F == 1 || (d_nodes && d_counters))), "NULL pointer");
    a.order = d_order; a.leaf_parent = (int32_t*)d_leaf_parent; a.nodes = d_nodes; a.tris = d_tris; a.counters = d_counters;
    return bvh_run<BVH_BOXES>(a, (int64_t)F, stream);
}

int perf_mesh_cast(const int32_t* d_nodes, const float* d_tris, uint64_t F, const float* d_rays_o, const float* d_rays_d, uint64_t R,
                   float t_min, float t_max, void* d_hits, void* stream)
{
    if (R == 0) return PERF_OK;
    CastArgs a;
    int rc = cast_fill(a, d_nodes, d_tris, F, t_min, t_max, d_hits); if (rc) return rc;
    PERF_CHECK_ARG(d_rays_o && d_rays_d, "NULL rays");
    PERF_CHECK_ARG(R < (1ull << 40), "%llu rays", (unsigned long long)R);
    a.o = d_rays_o; a.d = d_rays_d; a.R = (int64_t)R;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < a.R; ++i) cast_ray(a, i);
#else
    mesh_cast_kernel<<<(unsigned)((R + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

int perf_mesh_cast_pano(const int32_t* d_nodes, const float* d_tris, uint64_t F, const float* h_pose, int H, int W, int row0, int rows,
                        float t_min, float t_max, void* d_hits, void* stream)
{
    PERF_CHECK_ARG(h_pose, "NULL pose");
    PERF_CHECK_ARG(H > 0 && W > 0 && row0 >= 0 && rows >= 0 && row0 + rows <= H, "bad panorama window H=%d W=%d row0=%d rows=%d", H, W, row0, rows);
    if (rows == 0) return PERF_OK;
    CastArgs a;
    int rc = cast_fill(a, d_nodes, d_tris, F, t_min, t_max, d_hits); if (rc) return rc;
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) a.pose[3 * r + c] = h_pose[4 * r + c]; a.pose[9 + r] = h_pose[4 * r + 3]; }
    a.H = H; a.W = W; a.row0 = row0; a.rows = rows;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < W; ++x) cast_pixel(a, y, x);
#else
    const dim3 grid((unsigned)((W + PANO_TX - 1) / PANO_TX), (unsigned)((rows + PANO_TY - 1) / PANO_TY));
    mesh_cast_pano_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

static int shade_fill(ShadeArgs& a, const void* d_hits, const float* d_rays_d, uint64_t R, const float* d_vertices, uint64_t V,
                      const int32_t* d_faces, uint64_t F, const uint8_t* d_colors, const float* d_normals, const float* d_uv,
                      const uint8_t* d_texture, int T, float* d_rgb, float* d_distance, float* d_opacity, float* d_normal, uint8_t* d_back)
{
    PERF_CHECK_ARG(V < (1ull << 31) && F < (1ull << 30), "mesh of %llu vertices / %llu faces: needs V < 2^31 and F < 2^30",
                   (unsigned long long)V, (unsigned long long)F);
    PERF_CHECK_ARG(d_hits && d_rays_d && d_rgb && d_distance && d_opacity && d_normal && d_back, "NULL pointer");
    PERF_CHECK_ARG(F == 0 || (d_vertices && d_faces), "NULL vertices or faces");
    PERF_CHECK_ARG(!d_texture || (d_uv && T > 0 && T <= 65536), "texture without uv or of side %d", T);
    memset(&a, 0, sizeof(a));
    a.hits = (const float4*)d_hits; a.R = (int64_t)R; a.d = d_rays_d; a.pos = d_vertices; a.V = (int64_t)V; a.faces = d_faces;
    a.F = (int64_t)F; a.colors = d_colors; a.normals = d_normals; a.uv = d_uv; a.texture = d_texture; a.T = T;
    a.rgb = d_rgb; a.dist = d_distance; a.op = d_opacity; a.nrm = d_normal; a.back = d_back;
    return PERF_OK;
}

int perf_mesh_shade(const void* d_hits, const float* d_rays_d, uint64_t R, const float* d_vertices, uint64_t V, const int32_t* d_faces,
                    uint64_t F, const uint8_t* d_colors, const float* d_normals, const float* d_uv, const uint8_t* d_texture, int T,
                    float* d_rgb, float* d_distance, float* d_opacity, float* d_normal, uint8_t* d_back, void* stream)
{
    if (R == 0) return PERF_OK;
    ShadeArgs a;
    int rc = shade_fill(a, d_hits, d_rays_d, R, d_vertices, V, d_faces, F, d_colors, d_normals, d_uv, d_texture, T, d_rgb, d_distance,
                        d_opacity, d_normal, d_back);
    if (rc) return rc;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < a.R; ++i) shade_ray<false>(a, i);
#else
    mesh_shade_kernel<<<(unsigned)((R + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

int perf_mesh_shade_normal_texture(const void* d_hits, const float* d_rays_d, uint64_t R, const float* d_vertices, uint64_t V,
                                   const int32_t* d_faces, uint64_t F, const uint8_t* d_colors, const float* d_normals, const float* d_uv,
                                   const uint8_t* d_texture, const uint8_t* d_normal_texture, int T, float* d_rgb, float* d_distance,
                                   float* d_opacity, float* d_normal, uint8_t* d_back, void* stream)
{
    if (R == 0) return PERF_OK;
    PERF_CHECK_ARG(d_normal_texture && d_uv && T > 0 && T <= 65536, "normal texture without uv or of side %d", T);
    ShadeArgs a;
    int rc = shade_fill(a, d_hits, d_rays_d, R, d_vertices, V, d_faces, F, d_colors, d_normals, d_uv, d_texture, T, d_rgb, d_distance,
                        d_opacity, d_normal, d_back);
    if (rc) return rc;
    a.ntex = d_normal_texture;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < a.R; ++i) shade_ray<true>(a, i);
#else
    mesh_shade_normal_texture_kernel<<<(unsigned)((R + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

int perf_normal_texture_bake(const int32_t* d_nodes, const float* d_tris, const float* d_hi_vertices, uint64_t hi_V,
                             const int32_t* d_hi_faces, uint64_t hi_F, const float* d_hi_normals, const float* d_vertices, uint64_t V,
                             const int32_t* d_faces, uint64_t F, const float* d_normals, const float* d_uv, const int32_t* d_face,
                             const float* d_point, uint64_t N, float distance, uint8_t* d_texel, float* d_offset, void* stream)
{
    if (N == 0) return PERF_OK;
    PERF_CHECK_ARG(hi_V < (1ull << 31) && hi_F < (1ull << 30) && V < (1ull << 31) && F < (1ull << 30),
                   "meshes of %llu / %llu vertices and %llu / %llu faces: need V < 2^31 and F < 2^30", (unsigned long long)hi_V,
                   (unsigned long long)V, (unsigned long long)hi_F, (unsigned long long)F);
    PERF_CHECK_ARG(N < (1ull << 40), "%llu texels", (unsigned long long)N);
    PERF_CHECK_ARG(hi_F == 0 || (d_tris && (hi_F == 1 || d_nodes) && d_hi_vertices && d_hi_faces), "NULL high mesh or BVH");
    PERF_CHECK_ARG(F == 0 || (d_vertices && d_faces && d_uv), "NULL low mesh or uv");
    PERF_CHECK_ARG(d_face && d_point && d_texel && d_offset, "NULL pointer");
    PERF_CHECK_ARG(distance >= 0.0f && distance < INFINITY, "cast distance %g: needs a finite distance >= 0", (double)distance);
    BakeArgs a;
    memset(&a, 0, sizeof(a));
    a.nodes = d_nodes; a.tris = d_tris; a.hF = (int64_t)hi_F; a.hpos = d_hi_vertices; a.hfaces = d_hi_faces; a.hnormals = d_hi_normals;
    a.pos = d_vertices; a.faces = d_faces; a.normals = d_normals; a.uv = d_uv; a.face = d_face; a.point = d_point; a.N = (int64_t)N;
    a.dist = distance; a.texel = d_texel; a.offset = d_offset;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < a.N; ++i) bake_texel(a, i);
#else
    normal_texture_bake_kernel<<<(unsigned)((N + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

int perf_mesh_corner_tangents(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const float* d_normals,
                              const float* d_uv, float* d_tangents, void* stream)
{
    if (F == 0) return PERF_OK;
    PERF_CHECK_ARG(V < (1ull << 31) && F < (1ull << 30), "mesh of %llu vertices / %llu faces: needs V < 2^31 and F < 2^30",
                   (unsigned long long)V, (unsigned long long)F);
    PERF_CHECK_ARG(d_vertices && d_faces && d_uv && d_tangents, "NULL pointer");
    TangentArgs a;
    memset(&a, 0, sizeof(a));
    a.pos = d_vertices; a.faces = d_faces; a.normals = d_normals; a.uv = d_uv; a.F = (int64_t)F; a.out = d_tangents;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t f = 0; f < a.F; ++f) corner_tangents(a, f);
#else
    mesh_corner_tangents_kernel<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

#pragma GCC visibility pop
}
