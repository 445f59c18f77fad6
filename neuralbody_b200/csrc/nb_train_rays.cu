// nb_train_rays (include/neuralbody_b200.h): the training datasets' sample_ray_h36m / sample_ray, split 'train', on the
// device.  Three scans of the class map (scan_mask_bit, the scan nb_image_rays compacts with) give each class's row-major
// pixel list; one CTA per batch item then runs upstream's sampling rounds.  A candidate's ray is get_rays with
// nb_image_rays.cuh's roundings (camera_ray_d, K in its own dtype, R / T / o in float64) and get_near_far in float64, as
// numpy runs it on upstream's float64 rays.  No expression here may be contracted: every product and sum is an explicit _rn
// intrinsic.
#include <cub/block/block_scan.cuh>

#include "nb_image_rays.cuh"

namespace nb {
namespace {

constexpr int kSampleThreads = 256;
constexpr int kListThreads = 256;

// Philox4x32-10 (Salmon et al., SC'11) of the counter (k, round, item ^ key1.lo, key1.hi) under key0: the first 64 bits
__device__ __forceinline__ unsigned long long philox_u64(const unsigned long long (&key)[2], unsigned item, unsigned round,
                                                         unsigned k) {
    unsigned c0 = k, c1 = round, c2 = item ^ (unsigned)key[1], c3 = (unsigned)(key[1] >> 32);
    unsigned k0 = (unsigned)key[0], k1 = (unsigned)(key[0] >> 32);
    for (int r = 0; r < 10; ++r) {
        const unsigned lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
        const unsigned lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return ((unsigned long long)c1 << 32) | c0;
}

// get_rays at (x, y) in float64, then get_near_far (:54-69) in float64 on that one ray; -> mask_at_box
template <typename TK>
__device__ __forceinline__ bool train_ray(const ImageCam<TK, double>& c, const double* bnd, int x, int y, float (&of)[3],
                                          float (&df)[3], float& near, float& far) {
    double d[3];
    camera_ray_d(c, x, y, d);
    const double nrm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
    double t1[3], t2[3];
    for (int a = 0; a < 3; ++a) {
        double v = __ddiv_rn(d[a], nrm);
        if (v < 1e-5 && v > -1e-10) v = 1e-5;
        if (v > -1e-5 && v < 1e-10) v = -1e-5;
        const double tmin = __ddiv_rn(__dsub_rn(bnd[a], c.o[a]), v), tmax = __ddiv_rn(__dsub_rn(bnd[3 + a], c.o[a]), v);
        t1[a] = np_min(tmin, tmax);
        t2[a] = np_max(tmin, tmax);
        of[a] = __double2float_rn(c.o[a]);
        df[a] = __double2float_rn(d[a]);
    }
    const double tn = np_max(np_max(t1[0], t1[1]), t1[2]), tf = np_min(np_min(t2[0], t2[1]), t2[2]);
    near = __double2float_rn(__ddiv_rn(tn, nrm));
    far = __double2float_rn(__ddiv_rn(tf, nrm));
    return tn < tf;
}

struct Lists {
    const int* offset[3];   // the scans: exclusive prefix count of each class over the (B,H,W) map
    int* list[3];           // each class's pixels (index within the item), items one after another
    int* total[3];          // each class's count over the whole map
};

// the pixels of each class at their scanned offsets
__global__ void __launch_bounds__(kListThreads) train_lists_kernel(const unsigned char* __restrict__ cmap, int n, int hw,
                                                                   const __grid_constant__ Lists L) {
    const unsigned p = blockIdx.x * kListThreads + threadIdx.x;
    if (p >= (unsigned)n) return;
    const int m = cmap[p];
    for (int k = 0; k < 3; ++k) {
        const int bit = (m >> k) & 1, q = L.offset[k][p];
        if (bit) L.list[k][q] = (int)(p % (unsigned)hw);
        if (p == (unsigned)n - 1) *L.total[k] = q + bit;
    }
}

struct Sampler {
    nb_train_rays_args a;
    Lists L;
};

template <typename TK>
__global__ void __launch_bounds__(kSampleThreads) train_sample_kernel(const __grid_constant__ Sampler S) {
    using Scan = cub::BlockScan<int, kSampleThreads>;
    __shared__ typename Scan::TempStorage scan;
    const nb_train_rays_args& a = S.a;
    const int b = blockIdx.x, hw = a.H * a.W;
    const double* cam = a.cams + (size_t)b * NB_TRAIN_CAM_DOUBLES;
    ImageCam<TK, double> c;
    for (int k = 0; k < 9; ++k) { c.K_inv[k] = (TK)cam[k]; c.R[k] = cam[9 + k]; }
    for (int k = 0; k < 3; ++k) { c.T_[k] = cam[18 + k]; c.o[k] = cam[21 + k]; }
    const double* bnd = cam + 24;
    const int* list[3];
    int len[3];
    for (int k = 0; k < 3; ++k) {
        const int s0 = S.L.offset[k][(size_t)b * hw];
        const int s1 = b + 1 < a.B ? S.L.offset[k][(size_t)(b + 1) * hw] : *S.L.total[k];
        list[k] = S.L.list[k] + s0;
        len[k] = s1 - s0;
    }
    const bool replay = a.draws != nullptr;
    long long cursor = replay ? a.draw_offset[b] : 0;
    const long long draws_end = replay ? a.draw_offset[b + 1] : 0;
    const size_t slot0 = (size_t)b * a.n_rays;
    int sampled = 0, round = 0, status = NB_TRAIN_RAYS_OK;
    while (sampled < a.n_rays) {             // every value the loop reads is the block's: the threads leave together
        if (round == NB_TRAIN_RAYS_MAX_ROUNDS) { status = NB_TRAIN_RAYS_ROUNDS; break; }
        const int m = a.n_rays - sampled;
        const int n_body = (int)__dmul_rn((double)m, a.body_ratio), n_face = (int)__dmul_rn((double)m, a.face_ratio);
        const int n_rand = m - n_body - n_face;
        const int nf = len[1] > 0 ? n_face : 0;                    // upstream omits the face draws of an empty face list
        const int cands = n_body + nf + n_rand;
        if ((n_body > 0 && len[0] == 0) || (n_rand > 0 && len[2] == 0)) { status = NB_TRAIN_RAYS_EMPTY; break; }
        if (replay && (draws_end - cursor < cands)) { status = NB_TRAIN_RAYS_REPLAY; break; }
        bool bad = false;
        for (int k0 = 0; k0 < cands; k0 += kSampleThreads) {
            const int k = k0 + threadIdx.x;
            bool hit = false;
            float of[3], df[3], nr = 0.f, fr = 0.f;
            int pix = 0;
            if (k < cands) {
                const int cls = k < n_body ? 0 : (k < n_body + nf ? 1 : 2);   // selects, not indexing: no local memory
                const int* lst = cls == 0 ? list[0] : (cls == 1 ? list[1] : list[2]);
                const unsigned long long n = (unsigned long long)(cls == 0 ? len[0] : (cls == 1 ? len[1] : len[2]));
                unsigned long long idx;
                if (replay) {
                    const long long d = a.draws[cursor + k];
                    const bool out = d < 0 || (unsigned long long)d >= n;
                    bad |= out;
                    idx = out ? 0 : (unsigned long long)d;
                } else {
                    idx = __umul64hi(philox_u64(a.key, (unsigned)b, (unsigned)round, (unsigned)k), n);
                }
                if (!bad) {               // (a bad draw leaves the item's slots unspecified)
                    pix = lst[idx];
                    hit = train_ray(c, bnd, pix % a.W, pix / a.W, of, df, nr, fr);
                }
            }
            int pos, hits;
            Scan(scan).ExclusiveSum(hit ? 1 : 0, pos, hits);
            if (hit) {
                const size_t q = slot0 + sampled + pos;
                const float* px = a.image + ((size_t)b * hw + pix) * 3;
                for (int t = 0; t < 3; ++t) {
                    a.ray_o[q * 3 + t] = of[t];
                    a.ray_d[q * 3 + t] = df[t];
                    a.rgb[q * 3 + t] = px[t];
                }
                a.near[q] = nr;
                a.far[q] = fr;
                if (a.coord) a.coord[q] = pix;
            }
            sampled += hits;
            __syncthreads();                                       // the scan's storage is reused
        }
        if (__syncthreads_or(bad)) { status = NB_TRAIN_RAYS_REPLAY; break; }
        cursor += cands;
        ++round;
    }
    if (threadIdx.x == 0) {
        a.status[b] = status;
        if (a.rounds) a.rounds[b] = round;
    }
}

// H*W, or -1; B*H*W < 2^31 (the scans' int32 offsets)
int train_pixels(int B, int H, int W) {
    const int hw = image_rays_pixels(H, W);
    if (B < 1 || hw < 0 || (long long)B * hw >= (1LL << 31)) return -1;
    return B * hw;
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_train_rays_workspace_bytes(int B, int H, int W) {
    const int n = train_pixels(B, H, W);
    if (n < 0) return 0;
    const size_t sb = image_rays_scan_bytes(n);
    if (sb == 0) return 0;
    return 6 * align256((size_t)n * sizeof(int)) + align256(3 * sizeof(int)) + align256(sb);
}

int nb_train_rays(const nb_train_rays_args* a, void* stream) {
    static const char* who = "nb_train_rays";
    if (!a || !a->class_map || !a->image || !a->cams || !a->workspace || !a->ray_o || !a->ray_d || !a->near || !a->far ||
        !a->rgb || !a->status) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (!a->draws != !a->draw_offset) {
        set_error("%s: draws and draw_offset must both be set (replay) or both be NULL (Philox)", who);
        return NB_ERR_BAD_ARG;
    }
    const int n = train_pixels(a->B, a->H, a->W);
    if (n < 0) {
        set_error("%s: B, H and W must be >= 1 with B*H*W < 2^31 (got %d x %d x %d)", who, a->B, a->H, a->W);
        return NB_ERR_BAD_ARG;
    }
    if (a->n_rays < 1) {
        set_error("%s: n_rays must be >= 1 (got %d)", who, a->n_rays);
        return NB_ERR_BAD_ARG;
    }
    if (!(a->body_ratio >= 0.0 && a->face_ratio >= 0.0 && a->body_ratio + a->face_ratio <= 1.0)) {
        set_error("%s: the ratios must be >= 0 with body_ratio + face_ratio <= 1 (got %g, %g)", who, a->body_ratio,
                  a->face_ratio);
        return NB_ERR_BAD_ARG;
    }
    if ((a->k_kind != NB_SCALAR_F32 && a->k_kind != NB_SCALAR_F64) || a->rt_kind != NB_SCALAR_F64) {
        set_error("%s: k_kind must be NB_SCALAR_F32 or NB_SCALAR_F64 and rt_kind NB_SCALAR_F64 (got %d, %d)", who, a->k_kind,
                  a->rt_kind);
        return NB_ERR_BAD_ARG;
    }
    const size_t need = nb_train_rays_workspace_bytes(a->B, a->H, a->W);
    if (need == 0 || a->workspace_bytes < need) {
        set_error("%s: workspace_bytes too small (%zu < %zu)", who, a->workspace_bytes, need);
        return NB_ERR_BAD_ARG;
    }
    unsigned char* ws = (unsigned char*)a->workspace;
    const size_t arr = align256((size_t)n * sizeof(int));
    Sampler S;
    S.a = *a;
    for (int k = 0; k < 3; ++k) {
        S.L.offset[k] = (const int*)(ws + k * arr);
        S.L.list[k] = (int*)(ws + (3 + k) * arr);
        S.L.total[k] = (int*)(ws + 6 * arr) + k;
    }
    unsigned char* scratch = ws + 6 * arr + align256(3 * sizeof(int));
    size_t sb = need - (size_t)(scratch - ws);
    const cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaSuccess;
    for (int k = 0; k < 3 && e == cudaSuccess; ++k) e = scan_mask_bit(scratch, sb, a->class_map, k, (int*)S.L.offset[k], n, s);
    if (e == cudaSuccess) {
        const unsigned blocks = (unsigned)(((long long)n + kListThreads - 1) / kListThreads);
        train_lists_kernel<<<blocks, kListThreads, 0, s>>>(a->class_map, n, a->H * a->W, S.L);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        if (a->k_kind == NB_SCALAR_F32)
            train_sample_kernel<float><<<a->B, kSampleThreads, 0, s>>>(S);
        else
            train_sample_kernel<double><<<a->B, kSampleThreads, 0, s>>>(S);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // extern "C"
