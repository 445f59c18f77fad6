// nb_mesh_ply (include/neuralbody_b200.h): the binary PLY body of a triangle mesh on the device, the bytes
// neuralbody_b200.mcubes.Mesh.export writes after its header.  One launch over the body as 16-byte words:
//   - vertex blocks copy the (V,3) float64 array (the body's first 24 V bytes are its own bytes), two 8-byte loads per
//     16-byte store;
//   - face blocks stage the 13-byte records (uchar 3, three little-endian int32) of the faces that meet their run of
//     words in shared memory, then store whole 16-byte words, consecutive words by consecutive threads.  The first face
//     word also holds the last 8 vertex bytes when V is odd; the body's last word may be partial and is stored byte by
//     byte, so nothing past the body is written.
// The result record at the head of `out` (the body follows at NB_MESH_PLY_BODY_OFFSET, so one copy brings both back) is
// zeroed by a memset in stream order before the launch; a face index outside [0, max(V, 1)) (Mesh.export's bound) sets
// its status.
#include "nb_internal.h"

namespace nb {
namespace {

constexpr int kPlyThreads = 256;
constexpr int kPlyWordsPerThread = 4;
constexpr int kPlyBlockWords = kPlyThreads * kPlyWordsPerThread;   // 16 KB of body per block
constexpr int kPlyRecord = 13;

struct PlyGeom {
    long long nv, nf;
    long long base;          // 24 nv: where the face records start
    long long total;         // the body's bytes
    long long vwords;        // whole 16-byte words inside the vertex block
    long long words;         // 16-byte words of the body, the last one possibly partial
    unsigned vblocks;        // blocks of the vertex copy; the face blocks follow
};

inline PlyGeom ply_geom(long long nv, long long nf) {
    PlyGeom g;
    g.nv = nv;
    g.nf = nf;
    g.base = 24LL * nv;
    g.total = g.base + (long long)kPlyRecord * nf;
    g.vwords = g.base / 16;
    g.words = (g.total + 15) / 16;
    g.vblocks = (unsigned)((g.vwords + kPlyBlockWords - 1) / kPlyBlockWords);
    return g;
}

// store one 16-byte word of the body at word index w; the body's last word stops at `total`
__device__ __forceinline__ void store_word(unsigned char* body, long long w, long long total, uint4 v) {
    if (16 * w + 16 <= total) {
        reinterpret_cast<uint4*>(body)[w] = v;
    } else {
        const unsigned int part[4] = {v.x, v.y, v.z, v.w};
        for (long long j = 16 * w; j < total; ++j) {
            const int k = (int)(j - 16 * w);
            body[j] = (unsigned char)(part[k >> 2] >> (8 * (k & 3)));
        }
    }
}

__global__ void __launch_bounds__(kPlyThreads) mesh_ply_kernel(const __grid_constant__ nb_mesh_ply_args a,
                                                                const __grid_constant__ PlyGeom g) {
    __shared__ uint4 stage[kPlyBlockWords];
    unsigned char* body = a.out + NB_MESH_PLY_BODY_OFFSET;
    const unsigned long long* vbits = reinterpret_cast<const unsigned long long*>(a.vertices);
    const int t = threadIdx.x;
    if (blockIdx.x < g.vblocks) {
        const long long w0 = (long long)blockIdx.x * kPlyBlockWords;
#pragma unroll
        for (int k = 0; k < kPlyWordsPerThread; ++k) {
            const long long w = w0 + k * kPlyThreads + t;
            if (w < g.vwords) {
                const unsigned long long lo = __ldg(vbits + 2 * w), hi = __ldg(vbits + 2 * w + 1);
                reinterpret_cast<uint4*>(body)[w] =
                    make_uint4((unsigned)lo, (unsigned)(lo >> 32), (unsigned)hi, (unsigned)(hi >> 32));
            }
        }
        return;
    }
    // face blocks: words [w0, w1) of the body, bytes [b0, b1)
    const long long w0 = g.vwords + (long long)(blockIdx.x - g.vblocks) * kPlyBlockWords;
    const long long w1 = min(w0 + kPlyBlockWords, g.words);
    const long long b0 = 16 * w0, b1 = min(16 * w1, g.total);
    unsigned char* s = reinterpret_cast<unsigned char*>(stage);
    if (b0 < g.base && t < g.base - b0) {                 // the last 8 vertex bytes of an odd V
        const long long j = b0 + t;
        s[t] = (unsigned char)(vbits[j >> 3] >> (8 * (j & 7)));
    }
    const long long lim = g.nv > 1 ? g.nv : 1;
    const long long r0 = max(b0 - g.base, 0LL);              // record bytes of this block: [r0, r1)
    const long long r1 = b1 - g.base;
    const long long f0 = r0 / kPlyRecord, f1 = r1 > 0 ? (r1 + kPlyRecord - 1) / kPlyRecord : 0;
    bool bad = false;
    for (long long f = f0 + t; f < f1; f += kPlyThreads) {
        unsigned int rec[4];                              // the record's 13 bytes, little-endian, in words
        const long long* face = a.faces + 3 * f;
        unsigned int idx[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const long long v = __ldg(face + c);
            bad |= v < 0 || v >= lim;
            idx[c] = (unsigned int)v;                     // int32 of an in-range index; the file is not written otherwise
        }
        rec[0] = 3u | (idx[0] << 8);
        rec[1] = (idx[0] >> 24) | (idx[1] << 8);
        rec[2] = (idx[1] >> 24) | (idx[2] << 8);
        rec[3] = idx[2] >> 24;
        const long long at = g.base + kPlyRecord * f - b0;   // the record's first byte in the stage, may be < 0
#pragma unroll
        for (int k = 0; k < kPlyRecord; ++k) {
            const long long p = at + k;
            if (p >= 0 && p < b1 - b0) s[p] = (unsigned char)(rec[k >> 2] >> (8 * (k & 3)));
        }
    }
    if (bad) reinterpret_cast<nb_mesh_ply_result*>(a.out)->status = NB_MESH_PLY_FACE;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPlyWordsPerThread; ++k) {
        const int i = k * kPlyThreads + t;
        if (w0 + i < w1) store_word(body, w0 + i, g.total, stage[i]);
    }
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_mesh_ply_bytes(long long nv, long long nf) {
    if (nv < 0 || nf < 0 || nv >= (1LL << 31) || nf > (1LL << 40)) return 0;
    return (size_t)(24LL * nv + (long long)kPlyRecord * nf);
}

int nb_mesh_ply(const nb_mesh_ply_args* a, void* stream) {
    static const char* who = "nb_mesh_ply";
    if (!a || !a->out || (a->nv > 0 && !a->vertices) || (a->nf > 0 && !a->faces)) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->nv < 0 || a->nf < 0 || a->nf > (1LL << 40)) {
        set_error("%s: counts must be >= 0 with nf <= 2^40 (got nv = %lld, nf = %lld)", who, a->nv, a->nf);
        return NB_ERR_BAD_ARG;
    }
    if (a->nv >= (1LL << 31)) {
        set_error("%s: nv = %lld vertices: a PLY int32 index list holds < 2^31", who, a->nv);
        return NB_ERR_BAD_ARG;
    }
    if ((uintptr_t)a->out % 16 != 0 || (uintptr_t)a->vertices % 8 != 0 || (uintptr_t)a->faces % 8 != 0) {
        set_error("%s: out must be 16-byte aligned, vertices and faces 8-byte aligned", who);
        return NB_ERR_BAD_ARG;
    }
    const size_t need = NB_MESH_PLY_BODY_OFFSET + nb_mesh_ply_bytes(a->nv, a->nf);
    if (a->out_bytes < need) {
        set_error("%s: out_bytes too small (%zu < %zu)", who, a->out_bytes, need);
        return NB_ERR_BAD_ARG;
    }
    const cudaStream_t s = (cudaStream_t)stream;
    const PlyGeom g = ply_geom(a->nv, a->nf);
    cudaError_t e = cudaMemsetAsync(a->out, 0, sizeof(nb_mesh_ply_result), s);
    if (e == cudaSuccess && g.words > 0) {
        const unsigned fblocks = (unsigned)((g.words - g.vwords + kPlyBlockWords - 1) / kPlyBlockWords);
        mesh_ply_kernel<<<g.vblocks + fblocks, kPlyThreads, 0, s>>>(*a, g);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // extern "C"
