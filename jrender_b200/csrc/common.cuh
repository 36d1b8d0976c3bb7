// common.cuh -- shared definitions of the rasterizer kernels.
//
// Arithmetic contract: this translation unit set is compiled with -fmad=false
// (no a*b+c contraction), IEEE division and sqrt (nvcc defaults -prec-div=true,
// -prec-sqrt=true, -ftz=false).  Every +,-,*,/ below is therefore a separately
// rounded fp32 operation evaluated in the same order as the reference kernel
// source, which makes all discrete decisions of the rasterizer (border reject,
// inside tests, distance threshold, near/far reject, top-K membership, nearest
// face) bit-identical to oracle/softras_oracle.c.  Only expf() differs (<= 2 ulp).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define B200R_TILE 16          // fine tile edge in pixels (one CTA of 256 threads)
#define B200R_TILE_THREADS 256
#define B200R_BLOCK_W 8        // SoftRas forward block: 8x4 pixels, one warp, lane = row-major pixel index
#define B200R_BLOCK_H 4
#define B200R_MAX_COARSE_SIDE 16
#define B200R_LIST_CHUNK 512            // ids per chunk of the pooled coarse lists (a multiple of the forward's 128-entry filter pass)
#define B200R_LIST_CHUNK_SHIFT 9
#define B200R_LIST_IDS_PER_FACE 8       // pool budget: one partial chunk per bin + this many list entries per face

// Per-face record, 160 bytes, written once by the setup kernel and staged through
// shared memory by the raster kernels.  Replaces the reference's faces_info
// ([inv 9 | sym 9 | obt 3], cuda/soft_rasterize.py:190-192) plus the per-pixel
// recomputation of the face bounding box (check_border, :28-34), and carries the
// pre-computed refined reciprocals that make every per-face division MUFU-free
// (exact_math.cuh) and, for T == 1 surface textures, the face colour.
struct __align__(16) FaceRec {
    uint32_t rect_x;   // x0 | x1 << 16 : pixel columns passing check_border (inclusive)
    uint32_t rect_r;   // r0 | r1 << 16 : output rows passing check_border (inclusive, row 0 = top)
    uint32_t flags;    // bit k (k<3): face_obt[k]; bit 3: check_face_frontside;
                       // bit 4+k: midrange(z_k); bit 7+k: midrange(den_k)
    uint32_t face_id;  // index within the batch element
    float inv[9];      // face_inv  (:205-217)
    float v[9];        // x0 y0 z0 x1 y1 z1 x2 y2 z2
    float a0[9];       // a0[k][j] = sym[3k+j] - sym[3((k+1)%3)+j]   (:77-79, :128-130)
    float rz[3];       // rcp_refined(z_k)
    float rden[3];     // rcp_refined(den_k), den_k = a0[k][k] - a0[k][(k+1)%3]  (:81, :132)
    float col[3];      // textures[face][0][0..2] when T == 1 (surface), else 0
};
static_assert(sizeof(FaceRec) == 160, "FaceRec must be 160 bytes");
#define B200R_REC_UINT4 10  // 160 / 16

struct SoftRasParams {
    int B, nf, T, R, is, K;
    float near_, far_, eps, sigma, gamma, dist_eps;  // dist_eps = ln(1/dist_eps - 1)
    int dist_func, rgb_func, alpha_func, tex_type, double_side;
    int ntx;        // 16x16 tiles per image side (backward / NMR mapping)
    int fntx, fnty; // forward blocks (B200R_BLOCK_W x B200R_BLOCK_H) per image row / column
    int coarse_px;  // coarse bin edge in pixels (multiple of B200R_TILE)
    int ncs;        // coarse bins per image side
    int queue_len;    // persistent scheduler: entries of tile_order (one per forward block)
    int aa;           // backward: grad_soft_colors is the gradient of the 2x2-mean-pooled image [B,4,is/2,is/2] (anti-aliasing prologue)
};

// Device memory of one forward / backward pair, in two caller-allocated blocks (all offsets 256-byte aligned):
//   state     kept from the forward to the backward: the face records and the backward's gradient accumulator
//             (B*nf*208 bytes -- the reference keeps faces_info, 108 bytes per face, for the same purpose)
//   workspace transient scratch of the forward only (binning lists, tile queue): may be freed / reused as soon as the
//             forward has been enqueued
struct SoftRasWorkspace {
    FaceRec* recs;       // [B*nf]                                                               (state)
    float* gacc;         // [B*nf][12] backward gradient accumulator (3 x float4 per face)        (state)
    size_t state_bytes;
    uint2* rects;        // [B*nf]  (rect_x, rect_r) copy for the binning scans
    uint2* chunk_rects;  // [B*ceil(nf/256)] union rectangle of each run of 256 consecutive faces
    int* coarse_cnt;     // [B*ncs*ncs] list length; -1: the chunk pool ran out, the forward filters the whole face list for this bin
    int* chunk_table;    // [B*ncs*ncs][chunks_per_bin] pool chunk holding the list's k-th run of B200R_LIST_CHUNK ids
    int* coarse_pool;    // [pool_chunks][B200R_LIST_CHUNK] face ids, ascending within a list
    int chunks_per_bin, pool_chunks;
    int* counters;       // [256] scheduler state, zeroed per launch: [0] queue head, [1] pool cursor, [64..127] cost histogram, [128..191] scatter cursors
    int* tile_cost;      // [B*max_tiles] (pixel, face) pairs per forward block
    uint2* tile_order;   // [B*max_tiles] forward blocks, most expensive first: x = column | row << 16, y = image | (no face touches it) << 31
    size_t bytes;        // of the workspace block
};

static inline size_t b200r_align256(size_t x) { return (x + 255) & ~(size_t)255; }

static inline void b200r_geometry(int image_size, int* ntx, int* coarse_px, int* ncs) {
    const int nt = (image_size + B200R_TILE - 1) / B200R_TILE;
    int ctiles = (nt + B200R_MAX_COARSE_SIDE - 1) / B200R_MAX_COARSE_SIDE;  // tiles per coarse bin edge
    if (ctiles < 4) ctiles = 4;
    *ntx = nt;
    *coarse_px = ctiles * B200R_TILE;
    *ncs = (image_size + *coarse_px - 1) / *coarse_px;
}

static inline SoftRasWorkspace b200r_carve(void* state, void* base, int B, int nf, int image_size) {
    int ntx, cpx, ncs;
    b200r_geometry(image_size, &ntx, &cpx, &ncs);
    SoftRasWorkspace w;
    size_t off = 0;
    char* p = (char*)state;
    w.recs = (FaceRec*)(p + off);
    off += b200r_align256((size_t)B * nf * sizeof(FaceRec));
    w.gacc = (float*)(p + off);
    off += b200r_align256((size_t)B * nf * 12 * sizeof(float));
    w.state_bytes = off;
    off = 0;
    p = (char*)base;
    w.rects = (uint2*)(p + off);
    off += b200r_align256((size_t)B * nf * sizeof(uint2));
    w.chunk_rects = (uint2*)(p + off);
    off += b200r_align256((size_t)B * ((nf + 255) / 256) * sizeof(uint2));
    w.coarse_cnt = (int*)(p + off);
    off += b200r_align256((size_t)B * ncs * ncs * sizeof(int));
    // Coarse lists live in a pool of fixed-size chunks handed out by an atomic cursor while k_coarse_bin scans (capacity
    // nf per bin -- 160 MB at C3 -- would be the only overflow-proof layout without a host round trip for the totals).
    // A bin that finds the pool empty is flagged instead (coarse_cnt = -1) and the forward filters the whole face list
    // for its blocks: same faces, same order, only slower -- and lists that long mean every block holds most faces anyway.
    w.chunks_per_bin = (nf + B200R_LIST_CHUNK - 1) / B200R_LIST_CHUNK;
    {
        const size_t budget = (size_t)B * ncs * ncs + ((size_t)B * nf * B200R_LIST_IDS_PER_FACE + B200R_LIST_CHUNK - 1) / B200R_LIST_CHUNK;
        const size_t full = (size_t)B * ncs * ncs * w.chunks_per_bin;   // every list complete: never needs more than this
        const size_t n = budget < full ? budget : full;
        w.pool_chunks = (int)(n < (size_t)0x3fffff ? n : (size_t)0x3fffff);   // chunk << 9 stays inside 31 bits
    }
    w.chunk_table = (int*)(p + off);
    off += b200r_align256((size_t)B * ncs * ncs * w.chunks_per_bin * sizeof(int));
    w.coarse_pool = (int*)(p + off);
    off += b200r_align256((size_t)w.pool_chunks * B200R_LIST_CHUNK * sizeof(int));
    w.counters = (int*)(p + off);
    off += b200r_align256(256 * sizeof(int));
    // queue slots: the forward blocks of ntx x ntx 16x16 tiles
    const size_t max_tiles = (size_t)ntx * ntx * (B200R_TILE / B200R_BLOCK_W) * (B200R_TILE / B200R_BLOCK_H);
    w.tile_cost = (int*)(p + off);
    off += b200r_align256((size_t)B * max_tiles * sizeof(int));
    w.tile_order = (uint2*)(p + off);
    off += b200r_align256((size_t)B * max_tiles * sizeof(uint2));
    w.bytes = off;
    return w;
}

#ifdef __CUDACC__
// NDC coordinate of pixel index i (x: column; y: is-1-row), evaluated in double and
// rounded to float exactly like `(2. * xi + 1. - is) / is` (cuda/soft_rasterize.py:282-283).
//
// Evaluated as ONE fp32 division of the exact integers 2i + 1 - is and is: both are exactly representable, so the
// IEEE quotient is the correctly rounded value of the rational -- and so is the reference's double quotient rounded to
// float (a double rounding could only differ if the 53-bit quotient fell on a 24-bit rounding midpoint, which a ratio
// of integers below 2^14 cannot approach closer than 2^-38 relative).  Checked exhaustively for every image size up to
// the API limit of 4096 and every pixel index (tests/test_oracle_cpu.py).  The double division cost ~2 % of the forward.
__device__ __forceinline__ float b200r_pix_coord(int i, int is) {
    return __fdiv_rn((float)(2 * i + 1 - is), (float)is);
}
#endif
