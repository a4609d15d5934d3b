// tn_pairing.cuh -- from the sorted (t, face) keys of one ray to its records: the pairing stage of trace_rays
// (post_process_tetrahedra, src/optix/optix_trace_rays.cu:110-266, and the record emission of :216-225 with combine_indices :39-75).
// One warp per ray, keys and scratch in shared memory.  Used by k_trace<0> (tn_trace.cu) on keys gathered through the BVH or provided
// by a walk.  (Running it at the tail of the quad walk instead, each warp pairing the keys of its own rays that met eps-ties, was
// slower than the separate exact-stage launch: a warp with two or three such rays pairs them one after the other, while the exact
// stage gives every listed ray a warp of its own.)
#ifndef TN_PAIRING_CUH
#define TN_PAIRING_CUH
#include "tn_common.cuh"

namespace tn {
typedef unsigned long long u64;
#ifndef TN_EPS
#define TN_EPS 1e-6f  // optix_trace_rays.cu:8
#endif
namespace pairing {
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float key_t(u64 k) { return __uint_as_float((uint32_t)(k >> 32) & 0x7FFFFFFFu); }
__device__ __forceinline__ uint32_t key_face(u64 k) { return (uint32_t)k; }

// (t,u,v) of one ray/face pair, recomputed from the face's stored winding
__device__ __forceinline__ bool face_hit(const RaySetup &rs, const float *__restrict__ xyz, const uint4 tri, float &t, float &u,
                                         float &v) {
    const Sheared A = shear(rs, xyz[3 * (size_t)tri.x], xyz[3 * (size_t)tri.x + 1], xyz[3 * (size_t)tri.x + 2]);
    const Sheared B = shear(rs, xyz[3 * (size_t)tri.y], xyz[3 * (size_t)tri.y + 1], xyz[3 * (size_t)tri.y + 2]);
    const Sheared C = shear(rs, xyz[3 * (size_t)tri.z], xyz[3 * (size_t)tri.z + 1], xyz[3 * (size_t)tri.z + 2]);
    return tri_test(A, B, C, t, u, v);
}


static __device__ void bitonic_sort_keys(u64 *hits, uint32_t nh, int lane) {
    uint32_t P = 2;
    while (P < nh) P <<= 1;
    for (uint32_t i = nh + lane; i < P; i += 32) hits[i] = ~0ull;
    __syncwarp();
    for (uint32_t k = 2; k <= P; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t idx = lane; idx < (P >> 1); idx += 32) {
                const uint32_t i = ((idx & ~(j - 1)) << 1) | (idx & (j - 1));
                const uint32_t ij = i | j;
                const bool up = (i & k) == 0;
                const u64 a = hits[i], b = hits[ij];
                if ((a > b) == up) { hits[i] = b; hits[ij] = a; }
            }
            __syncwarp();
        }
    }
}

// literal post_process_tetrahedra (optix_trace_rays.cu:110-266) on the sorted keys.
// key bit 63 plays hit_distances[].y (the "marked once" flag); face == TN_EMPTY plays t[j] == empty.
// Every emitted record pairs position j with position j+1 of the array AFTER the swap of :229-235,
// so only the list of j's is produced; the caller emits (hits[j], hits[j+1]).
// The two loop bodies are functions of j so that the whole-array form (post_process_serial, one lane) and the windowed form
// (post_process_windows) execute the same statements.
constexpr u64 KEY_MARK = 1ull << 63;
// dedupe phase, body of the loop over j (optix_trace_rays.cu:124-159); key[j] is not empty, j + 1 < n
__device__ __forceinline__ void dedupe_one(u64 *key, const uint2 *tts, uint32_t n, uint32_t j) {
    const float dn = key_t(key[j]);
    bool clear_self = false;
    for (uint32_t off = 1; j + off < n && (key_face(key[j + off]) == TN_EMPTY || fabsf(__fsub_rn(key_t(key[j + off]), dn)) < TN_EPS); ++off) {
        uint32_t cell;
        if (key_face(key[j + off]) != TN_EMPTY && common_tet(tts[j], tts[j + off], cell)) {
            if (key_face(key[j]) != key_face(key[j + off])) clear_self = true;
            if (key[j + off] & KEY_MARK) key[j + off] |= 0xFFFFFFFFull;  // already marked once -> delete
            else key[j + off] |= KEY_MARK;
        }
    }
    if (clear_self && (key[j] & KEY_MARK)) key[j] |= 0xFFFFFFFFull;
    key[j] &= ~KEY_MARK;
}
// pairing phase, body of the loop over j (optix_trace_rays.cu:161-258); key[j] is not empty.  Returns whether record (j, j+1) is
// emitted; rd / wr are raised to the largest index the body read / wrote (the swap).
__device__ __forceinline__ bool pair_one(u64 *key, uint2 *tts, uint32_t n, uint32_t j, uint32_t &rd, uint32_t &wr) {
    const uint2 orig = tts[j];
    float dn = key_t(key[j]);
    uint32_t real_offset = 1, off = 1;
    bool emitted = false;
    for (; j + off < n && (real_offset < 3 || key_face(key[j + off]) == TN_EMPTY || fabsf(__fsub_rn(key_t(key[j + off]), dn)) < TN_EPS); ++off) {
        if (key_face(key[j + off]) == TN_EMPTY) continue;
        uint32_t cell;
        if (common_tet(orig, tts[j + off], cell)) {
            const bool out = fabsf(__fsub_rn(key_t(key[j]), key_t(key[j + off]))) >= TN_EPS;
            if (off > 1) {
                const u64 tk = key[j + off]; key[j + off] = key[j + 1]; key[j + 1] = tk;
                const uint2 tc = tts[j + off]; tts[j + off] = tts[j + 1]; tts[j + 1] = tc;
                wr = max(wr, j + off);
            }
            emitted = out;
            break;
        }
        dn = key_t(key[j + off]);
        real_offset++;
    }
    rd = max(rd, min(j + off, n - 1));
    return emitted;
}
// the whole array on one lane
static __device__ uint32_t post_process_serial(u64 *key, uint2 *tts, uint32_t n, uint16_t *emit) {
    for (uint32_t j = 0; j + 1 < n; ++j)
        if (key_face(key[j]) != TN_EMPTY) dedupe_one(key, tts, n, j);
    uint32_t jc = 0, rd = 0, wr = 0;
    for (uint32_t j = 0; j < n; ++j)
        if (key_face(key[j]) != TN_EMPTY && pair_one(key, tts, n, j, rd, wr)) emit[jc++] = (uint16_t)j;
    return jc;
}

// Windowed form: the same statements, executed only where they can do something.  Call position j "linked" to j+1 when the two hits
// are closer than eps or share no tetrahedron.  Away from the runs of links the literal algorithm is the identity pairing: the dedupe
// body touches nothing (its scan stops at the first hit >= eps away), the pairing body finds its partner at offset 1, emits, swaps
// nothing.  Around a run of links s..e the dedupe phase marks / deletes only hits within eps of one another (inside the run) and the
// pairing body of j in [s-1, e] reads at most up to e+2 (real_offset < 3) and swaps inside that range -- so the bodies are run for the
// windows [s-1, e+2] only, IN ORDER and on ONE lane like the literal loops, and the pairing loop keeps going past a window for as long
// as its swaps reached (a swapped position is no longer "clean"; such cascades can run to the end of the ray).  The links, the
// windows, the default decisions and the compaction of the emitted j's are computed by the whole warp.  A typical ray of the walk's
// exact list has 1-2 windows of ~5 positions among ~170 hits.  mask = 3 * ceil(n / 32) words of shared memory; returns the number
// of records, their j's in emit[].
__device__ __forceinline__ uint32_t next_set_bit(const uint32_t *W, uint32_t nw, uint32_t from, uint32_t none) {
    for (uint32_t c = from >> 5; c < nw; ++c) {
        uint32_t o = W[c];
        if (c == (from >> 5)) o &= ~0u << (from & 31u);
        if (o) return (c << 5) + (uint32_t)__ffs(o) - 1u;
    }
    return none;
}
__device__ __forceinline__ uint32_t next_clear_bit(const uint32_t *W, uint32_t nw, uint32_t from, uint32_t none) {
    for (uint32_t c = from >> 5; c < nw; ++c) {
        uint32_t z = ~W[c];
        if (c == (from >> 5)) z &= ~0u << (from & 31u);
        if (z) return (c << 5) + (uint32_t)__ffs(z) - 1u;
    }
    return none;
}
static __device__ __noinline__ uint32_t post_process_windows(u64 *key, uint2 *tts, uint32_t n, uint16_t *emit, uint32_t *mask, int lane) {
    const uint32_t nw = (n + 31) >> 5;
    uint32_t *L = mask, *W = mask + nw, *E = mask + 2 * nw;  // links; window / processed positions; emitted positions
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t j = base + lane;
        bool link = false;
        if (j + 1 < n) {
            uint32_t cell;
            link = fabsf(__fsub_rn(key_t(key[j + 1]), key_t(key[j]))) < TN_EPS || !common_tet(tts[j], tts[j + 1], cell);
        }
        const uint32_t w = __ballot_sync(FULL, link);
        if (lane == 0) { L[base >> 5] = w; E[base >> 5] = 0u; }
    }
    __syncwarp();
    for (uint32_t c = lane; c < nw; c += 32) {  // W[j] = OR of link[j-3 .. j+1]
        const uint32_t l = L[c], lp = c ? L[c - 1] : 0u, ln = c + 1 < nw ? L[c + 1] : 0u;
        uint32_t w = l | (l >> 1) | (ln << 31) | (l << 1) | (lp >> 31) | (l << 2) | (lp >> 30) | (l << 3) | (lp >> 29);
        if (c == nw - 1 && (n & 31u)) w &= (1u << (n & 31u)) - 1u;  // positions >= n: clear (so that every run ends inside the array)
        W[c] = w;
    }
    __syncwarp();
    if (lane == 0) {
        // dedupe phase (the loop of :124-159) over the windows
        for (uint32_t ws = next_set_bit(W, nw, 0, n); ws < n;) {
            const uint32_t we = min(next_clear_bit(W, nw, ws, n), n) - 1u;  // last position of the run
            for (uint32_t j = ws; j <= we && j + 1 < n; ++j)
                if (key_face(key[j]) != TN_EMPTY) dedupe_one(key, tts, n, j);
            ws = next_set_bit(W, nw, we + 1, n);
        }
        // pairing phase (the loop of :161-258) over the windows and whatever their swaps reach
        for (uint32_t ws = next_set_bit(W, nw, 0, n); ws < n;) {
            const uint32_t we = min(next_clear_bit(W, nw, ws, n), n) - 1u;
            uint32_t lim = we, rd = 0, wr = 0;
            for (uint32_t j = ws; j <= lim && j < n; ++j) {
                const bool em = key_face(key[j]) != TN_EMPTY && pair_one(key, tts, n, j, rd, wr);
                lim = max(lim, wr);
                if (j > we) W[j >> 5] |= 1u << (j & 31u);  // processed here although outside the window
                if (em) E[j >> 5] |= 1u << (j & 31u);
            }
            ws = next_set_bit(W, nw, lim + 1, n);
        }
    }
    __syncwarp();
    uint32_t jc = 0;
    for (uint32_t base = 0; base < n; base += 32) {  // compact: processed positions as decided above, the others pair with their successor
        const uint32_t j = base + lane;
        const uint32_t w = W[base >> 5], e = E[base >> 5];
        const bool em = ((w >> lane) & 1u) ? ((e >> lane) & 1u) != 0u : (j + 1 < n);
        const uint32_t m = __ballot_sync(FULL, em);
        if (em) emit[jc + __popc(m & ((1u << lane) - 1u))] = (uint16_t)j;
        jc += __popc(m);
    }
    return jc;
}

// keys that are sorted up to a few local inversions (the walk's keys: ties only): odd-even transposition passes, bitonic if they do
// not suffice.  Keys are distinct, so every correct sort gives the same array.
static __device__ __noinline__ void sort_nearly_sorted(u64 *hits, uint32_t nh, int lane) {
    for (int pass = 0; pass < 5; ++pass) {
        bool inv = false;
        for (uint32_t j = lane; j + 1 < nh; j += 32) inv |= hits[j] > hits[j + 1];
        if (!__any_sync(FULL, inv)) return;
        if (pass == 4) break;
        for (uint32_t par = 0; par < 2; ++par) {
            __syncwarp();
            for (uint32_t i = 2 * lane + par; i + 1 < nh; i += 64) {
                const u64 a = hits[i], b = hits[i + 1];
                if (a > b) { hits[i] = b; hits[i + 1] = a; }
            }
        }
        __syncwarp();
    }
    bitonic_sort_keys(hits, nh, lane);
}

// where the records of a ray go
struct PairOut {
    uint32_t *cells, *verts;
    float *bary, *dist;
};

// hits[0..nh) sorted by (t, face) -> the records of the ray whose first record is row `row`; returns their number.  Warp-collective.
// tts: nh uint2, emit: nh uint16, mask: 3 * ceil(nh / 32) words for the windowed pairing or nullptr (single-lane literal form).
__device__ __forceinline__ uint32_t pair_and_emit(u64 *hits, uint2 *tts, uint16_t *emit, uint32_t *mask, uint32_t nh, const uint2 *__restrict__ tt,
                                                  const uint4 *__restrict__ tri, const float *__restrict__ xyz, const RaySetup &rs, size_t row,
                                                  const PairOut &out, int lane) {
    uint32_t jc = 0;
    if (nh >= 2) {
        for (uint32_t j = lane; j < nh; j += 32) tts[j] = __ldg(tt + key_face(hits[j]));
        __syncwarp();
        // Parallel pairing whenever the literal algorithm reduces to "pair consecutive hits, skip crossings shorter
        // than eps": every consecutive pair shares a tetrahedron, and a crossing shorter than eps is ISOLATED
        // (strictly increasing t, both neighbouring crossings >= eps) -- then the dedupe phase marks and unmarks
        // without deleting (optix_trace_rays.cu:124-159) and the pairing phase skips that record (:208).
        bool ok = true;
        for (uint32_t j = lane; j + 1 < nh; j += 32) {
            uint32_t cell;
            const float tj = key_t(hits[j]), tn = key_t(hits[j + 1]);
            if (!common_tet(tts[j], tts[j + 1], cell)) ok = false;
            if (fabsf(__fsub_rn(tn, tj)) < TN_EPS) {
                if (!(tn > tj)) ok = false;
                if (j > 0 && fabsf(__fsub_rn(tj, key_t(hits[j - 1]))) < TN_EPS) ok = false;
                if (j + 2 < nh && fabsf(__fsub_rn(key_t(hits[j + 2]), tn)) < TN_EPS) ok = false;
            }
        }
        if (__all_sync(FULL, ok)) {
            for (uint32_t base = 0; base + 1 < nh; base += 32) {  // compact the emitted pair indices
                const uint32_t j = base + lane;
                const bool em = j + 1 < nh && !(fabsf(__fsub_rn(key_t(hits[j + 1]), key_t(hits[j]))) < TN_EPS);
                const uint32_t mask = __ballot_sync(FULL, em);
                if (em) emit[jc + __popc(mask & ((1u << lane) - 1u))] = (uint16_t)j;
                jc += __popc(mask);
            }
        } else {
            // rays with eps-ties that are not isolated (5-6 % of a batch): the literal algorithm restricted to the windows around
            // the ties (when the caller has room for the mask words)
            bool windowed = false;
            if (mask != nullptr) {
                jc = post_process_windows(hits, tts, nh, emit, mask, lane);
                windowed = true;
            }
            if (!windowed) {
                if (lane == 0) jc = post_process_serial(hits, tts, nh, emit);
                jc = __shfl_sync(FULL, jc, 0);
            }
        }
        __syncwarp();
    }
    for (uint32_t r = lane; r < jc; r += 32) {
        const uint32_t j = (uint32_t)emit[r];
        const uint32_t f0 = key_face(hits[j]), f1 = key_face(hits[j + 1]);
        const uint4 tr0 = __ldg(tri + f0), tr1 = __ldg(tri + f1);
        float t0, u0, v0, t1, u1, v1;
        face_hit(rs, xyz, tr0, t0, u0, v0);
        face_hit(rs, xyz, tr1, t1, u1, v1);
        uint32_t cell = TN_EMPTY;
        common_tet(tts[j], tts[j + 1], cell);
        // combine_indices (optix_trace_rays.cu:39-75)
        const float b00 = __fsub_rn(__fsub_rn(1.0f, u0), v0);
        const float r2[3] = {__fsub_rn(__fsub_rn(1.0f, u1), v1), u1, v1};
        const uint32_t id1[3] = {tr0.x, tr0.y, tr0.z}, id2[3] = {tr1.x, tr1.y, tr1.z};
        float o2[3] = {0.f, 0.f, 0.f};
        uint32_t newv = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            bool was = false;
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                if (!was && id1[q] == id2[i]) { o2[q] = r2[i]; was = true; }
            }
            if (!was) newv = id2[i];
        }
        const size_t g = row + r;
        out.cells[g] = cell;
        reinterpret_cast<uint4 *>(out.verts)[g] = make_uint4(newv, tr0.x, tr0.y, tr0.z);
        float2 *bp = reinterpret_cast<float2 *>(out.bary + 6 * g);
        bp[0] = make_float2(b00, u0);
        bp[1] = make_float2(v0, o2[0]);
        bp[2] = make_float2(o2[1], o2[2]);
        reinterpret_cast<float2 *>(out.dist)[g] = make_float2(t0, t1);
    }
    return jc;
}

}  // namespace pairing
}  // namespace tn
#endif
