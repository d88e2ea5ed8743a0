// ringpacking.cu -- RLWE ring packing on the device, for a BATCH of ciphertexts sharing one set of Galois keys, on a single ring
// degree (the reference's MinLogN == MaxLogN):
//   RingPackingEvaluator.Expand   core/rlwe/ring_packing.go:457-571   (one ciphertext -> N / 2^logGap one-coefficient ciphertexts)
//   RingPackingEvaluator.Pack     core/rlwe/ring_packing.go:600-770   (the inverse tree)
// Both trees are data-independent, so the host plans every step (and looks up every key) before any device work. At each step of
// either tree every key switch uses the same Galois element: the ciphertexts to key-switch are laid out as one uniformly strided
// block and go through ONE gadget product per step per batch_chunk() of them, so the key is read once per sub-batch instead of
// once per ciphertext. The additions, the multiplications by X^k and the automorphisms around each step are two fused passes:
//   pack_pre_kernel     a' = a + b X^k, t = a - b X^k (or the one-sided cases), with the pre-scaling folded into the first step;
//   pack_post_kernel /  a' +- phi(t + ks) gathered through the in-thread AutomorphismNTTIndex;
//   expand_post_kernel  c0 + phi(c0 + ks) and (c0 - phi(c0 + ks)) X^-n.
// Every output is a canonical residue that depends on its inputs only through residue classes, so the results equal the
// reference bit for bit (DESIGN 3.4; tests/test_gpu_ringpacking.py vs oracle/ringpacking.py).
#include <algorithm>
#include <string>
#include <vector>
#include "capi_common.h"
#include "composite.h"
#include "modarith.cuh"
#include "xpow.cuh"

namespace lgpu {

// ---------------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ u64 rp_sub(u64 a, u64 b, u64 q) { return a >= b ? a - b : a + q - b; }

// one tree step of Pack: the pairs (jx, jy) that hold at least one ciphertext
enum { PAIR_AB = 0, PAIR_A = 1, PAIR_B = 2 };
struct Pair { int a, b, dst, kind; };     // a / b: source positions (-1 = nil), dst: work slot the pair's result lives in

struct PackPreParams {
    const LimbConst* limbs;
    const Pair* pairs; int batch, e0, m;      // elements e0 .. e0 + m - 1 of the step; element e = pair e / batch, entry e % batch
    const u64* src; size_t src_ss, src_bs;    // a / b of pair element (p, b) at src + pos * src_ss + b * src_bs (step 0: the inputs)
    u64* work; size_t work_ss;                // slot-major work block: slot s of batch entry b at work + s * work_ss + b * cs
    u64* t;                                   // key-switch staging of the chunk, [m][2][nq][N]
    size_t cs;                                // component stride (level + 1) * N
    u64 k; int lg; u64 mask2n; int n;         // X^k, log2 N, 2N - 1, N
    int scale;                                // first step: multiply a and b by sc[r] (plain, Shoup sc_sh[r])
    u64 sc[kMaxRows], sc_sh[kMaxRows];
};
// both present: work[dst] = a + b X^k, t = a - b X^k;  b only: work[dst] = t = b X^k;  a only: work[dst] = t = a
// (ring_packing.go:700-722, :665-684 for the scaling)
__global__ void __launch_bounds__(256) pack_pre_kernel(PackPreParams p) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const int r = blockIdx.y;
    const LimbConst L = p.limbs[r];
    const u64 q = L.q;
    const u64 odd = 2 * (__brevll((u64)j) >> (64 - p.lg)) + 1;
    const size_t ro = (size_t)r * p.n + j;
    for (int z = blockIdx.z; z < p.m; z += gridDim.z) {
        const int e = p.e0 + z;
        const Pair pr = p.pairs[e / p.batch];
        const size_t b = (size_t)(e % p.batch);
        u64* w = p.work + (size_t)pr.dst * p.work_ss + b * 2 * p.cs + ro;
        u64* t = p.t + (size_t)z * 2 * p.cs + ro;
        for (int comp = 0; comp < 2; comp++) {
            const size_t co = comp * p.cs;
            u64 a = 0, x = 0;
            if (pr.kind != PAIR_B) {
                a = p.src[(size_t)pr.a * p.src_ss + b * p.src_bs + co + ro];
                if (p.scale) a = cred(a * p.sc[r] - __umul64hi(a, p.sc_sh[r]) * q, q);
            }
            if (pr.kind != PAIR_A) {
                x = p.src[(size_t)pr.b * p.src_ss + b * p.src_bs + co + ro];
                if (p.scale) x = cred(x * p.sc[r] - __umul64hi(x, p.sc_sh[r]) * q, q);
                x = mul_xpow(x, p.k, odd, L, p.lg, p.mask2n);
            }
            if (pr.kind == PAIR_AB) { w[co] = cred(a + x, q); t[co] = rp_sub(a, x, q); }
            else if (pr.kind == PAIR_B) { w[co] = x; t[co] = x; }
            else { w[co] = a; t[co] = a; }
        }
    }
}

struct PackPostParams {
    const LimbConst* limbs;
    const Pair* pairs; int batch, e0, m;        // elements e0 .. e0 + m - 1 of the step
    const u64* t; const u64* ks; size_t ks_cs;  // t: the chunk's staging [m][2][nq][N]; ks: GadgetProduct(t[1]), [2][m][nq][N]
    u64* work; size_t work_ss, cs;
    u64 galEl, mask2n; int lg, n;
};
// work[dst] = base +- phi(t + ks) (ring_packing.go:724-765): + for the pairs holding a, - for b only. In place: each thread reads
// base at its own position, the gather reads only t and ks.
__global__ void __launch_bounds__(256) pack_post_kernel(PackPostParams p) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const int r = blockIdx.y;
    const u64 q = p.limbs[r].q;
    const size_t idx = auto_index(j, p.galEl, p.mask2n, p.lg), ro = (size_t)r * p.n;
    for (int z = blockIdx.z; z < p.m; z += gridDim.z) {
        const int e = p.e0 + z;
        const Pair pr = p.pairs[e / p.batch];
        const size_t b = (size_t)(e % p.batch);
        const u64* t0 = p.t + (size_t)z * 2 * p.cs + ro;
        const u64* k0 = p.ks + (size_t)z * p.cs + ro;
        u64* w0 = p.work + (size_t)pr.dst * p.work_ss + b * 2 * p.cs + ro;
        const u64 u0 = cred(t0[idx] + k0[idx], q), u1 = k0[p.ks_cs + idx];
        if (pr.kind == PAIR_B) {
            w0[j] = rp_sub(w0[j], u0, q);
            w0[p.cs + j] = rp_sub(w0[p.cs + j], u1, q);
        } else {
            w0[j] = cred(w0[j] + u0, q);
            w0[p.cs + j] = cred(w0[p.cs + j] + u1, q);
        }
    }
}

struct ExpandPostParams {
    const LimbConst* limbs;
    int batch, e0, m, cnt;                      // elements e0 .. e0 + m - 1 of the step; cnt = inputs per batch entry
    const u64* in;                              // c0 of element e = s * batch + b at in + e * 2 * cs (slot-major)
    const u64* ks; size_t ks_cs;                // GadgetProduct(c0[1]) for these elements, [2][m][nq][N]
    u64* out; size_t out_ss, out_bs, cs;        // slot s of batch entry b at out + s * out_ss + b * out_bs
    int odd;                                    // n >= gap: also write slot s + cnt
    u64 galEl, kinv, mask2n; int lg, n;         // kinv = 2N - n (X^-n)
};
// even = c0 + phi(c0 + ks), odd = (c0 - phi(c0 + ks)) X^-n (ring_packing.go:526-559). Not in place: the gather reads c0 elsewhere.
__global__ void __launch_bounds__(256) expand_post_kernel(ExpandPostParams p) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const int r = blockIdx.y;
    const LimbConst L = p.limbs[r];
    const u64 q = L.q;
    const size_t idx = auto_index(j, p.galEl, p.mask2n, p.lg), ro = (size_t)r * p.n;
    const u64 slot_odd = 2 * (__brevll((u64)j) >> (64 - p.lg)) + 1;
    for (int z = blockIdx.z; z < p.m; z += gridDim.z) {
        const int e = p.e0 + z;
        const size_t s = (size_t)(e / p.batch), b = (size_t)(e % p.batch);
        const u64* c0 = p.in + (size_t)e * 2 * p.cs + ro;
        const u64* k0 = p.ks + (size_t)z * p.cs + ro;
        const u64 u0 = cred(c0[idx] + k0[idx], q), u1 = k0[p.ks_cs + idx];
        const u64 x0 = c0[j], x1 = c0[p.cs + j];
        u64* ev = p.out + s * p.out_ss + b * p.out_bs + ro;
        ev[j] = cred(x0 + u0, q);
        ev[p.cs + j] = cred(x1 + u1, q);
        if (p.odd) {
            u64* od = ev + (size_t)p.cnt * p.out_ss;
            od[j] = mul_xpow(rp_sub(x0, u0, q), p.kinv, slot_odd, L, p.lg, p.mask2n);
            od[p.cs + j] = mul_xpow(rp_sub(x1, u1, q), p.kinv, slot_odd, L, p.lg, p.mask2n);
        }
    }
}

namespace {

constexpr unsigned kMaxGridZ = 65535;

int log2_nthroot_half(const Ctx* c) {
    int lg = 0;
    while ((1ull << (lg + 1)) < c->nthroot) lg++;
    return lg;
}
u64 shoup(u64 w, u64 q) { return (u64)(((unsigned __int128)w << 64) / q); }

// a key gadget_product accepts at `level` (the reference's Automorphism -> GadgetProduct), looked up before any device work
int lookup(const Ctx* c, const GaloisKeySet& ks, int level, u64 g, const GadgetCt*& out) {
    out = ks.find(g);
    if (!out) return -1;
    if (check_evk(c, level, *out)) return -1;
    if (out->levelP > 0 && out->pw2 != 0) { set_error("BaseTwoDecomposition != 0 requires levelP <= 0"); return -1; }
    return 0;
}

// ct_in scaled by 2^-s mod Q_level (MulScalarBigint, canonical per limb), MForm'd scalars for MULSCALARMONTGOMERY
std::vector<u64> pow2_inv_mform(const Ctx* c, int nq, int s) {
    std::vector<u64> v(nq);
    for (int i = 0; i < nq; i++) v[i] = h_mform(h_invmod(h_powmod(2, (u64)s, c->Q[i]), c->Q[i]), c->Q[i]);
    return v;
}

// one gadget product per batch_chunk() of the m elements of a step: `pre(e0, nb)` returns the chunk's ciphertexts as one block of
// nb consecutive [2][nq][N] ciphertexts (nullptr on error), `post(e0, nb, ks)` consumes the key-switched chunk
template <class Pre, class Post>
int keyswitch_chunks(const Ctx* c, int level, int m, const GadgetCt& key, u64* ks, cudaStream_t st, Pre pre, Post post) {
    const size_t N = c->N, nq = level + 1, cs = nq * N;
    const int ch = batch_chunk();
    for (int e0 = 0; e0 < m; e0 += ch) {
        const int nb = std::min(ch, m - e0);
        const u64* block = pre(e0, nb);
        if (!block) return -1;
        if (gadget_product(c, level, CSpan{block + cs, N, 2 * cs}, key, Span{ks, N, cs}, Span{ks + (size_t)nb * cs, N, cs}, nb, st))
            return -1;
        if (post(e0, nb, ks)) return -1;
    }
    return 0;
}

// ---- Expand ---------------------------------------------------------------------------------------------------------
struct ExpandStep { int cnt; bool odd; u64 galEl; const GadgetCt* key; };

std::vector<ExpandStep> expand_schedule(const Ctx* c, int log_gap) {
    std::vector<ExpandStep> s;
    const long long gap = 1ll << log_gap;
    for (int i = 0; i < c->logN; i++) {
        const long long n = 1ll << i;
        ExpandStep e;
        e.odd = n >= gap;                                   // j + n / gap > 0 (:536)
        e.cnt = e.odd ? (int)(n / gap) : 1;                 // j = 0, gap, ..., < n
        e.galEl = (u64)(c->N / n + 1);
        e.key = nullptr;
        s.push_back(e);
    }
    return s;
}

int expand_run(const Ctx* c, int level, const u64* ct_in, bool is_ntt, int log_gap, const std::vector<ExpandStep>& sched, u64* ct_out, int B,
               cudaStream_t st) {
    const size_t N = c->N, nq = level + 1, cs = nq * N, ct = 2 * cs;
    const int d = (int)sched.size(), S = c->N >> log_gap;
    const int ch = batch_chunk();
    const size_t a_cts = (size_t)std::max(1, S / 2) * B;
    int max_m = 0;
    for (const ExpandStep& s : sched) max_m = std::max(max_m, std::min(ch, s.cnt * B));
    Scratch buf;
    if (buf.alloc(a_cts * ct + (size_t)max_m * ct, st)) return -1;
    u64* A = buf.p;
    u64* ks = buf.p + a_cts * ct;
    // step i reads X[i] (slot-major) and writes X[i+1]; X[d] is ct_out, the others alternate between A and ct_out's own memory used
    // as a slot-major scratch (step i < d - 1 writes at most S / 4 slots per batch entry, ct_out holds S)
    auto X = [&](int i) -> u64* { return ((d - 1 - i) & 1) ? ct_out : A; };
    const int lg = log2_nthroot_half(c);
    const std::vector<u64> sc = pow2_inv_mform(c, (int)nq, c->logN);
    u64* x0 = X(0);
    if (launch_vecop(c, rows_range(0, 0, (int)nq), LGPU_OP_MULSCALARMONTGOMERY, CSpan{ct_in, N, cs}, CSpan{nullptr, 0, 0}, Span{x0, N, cs}, 2 * B,
                     sc.data(), nullptr, 0, 0, c->N, st)) return -1;
    if (!is_ntt && launch_ntt(c, rows_range(0, 0, (int)nq), CSpan{x0, N, cs}, Span{x0, N, cs}, 2 * B, NTT_CANONICAL, st)) return -1;
    for (int i = 0; i < d; i++) {
        const ExpandStep& s = sched[i];
        const bool last = i == d - 1;
        ExpandPostParams p;
        p.limbs = c->d_limbs; p.batch = B; p.cnt = s.cnt; p.in = X(i); p.ks_cs = 0; p.out = X(i + 1);
        p.out_ss = last ? ct : (size_t)B * ct; p.out_bs = last ? (size_t)S * ct : ct; p.cs = cs; p.odd = s.odd ? 1 : 0;
        p.galEl = s.galEl; p.kinv = 2 * (u64)c->N - ((u64)1 << i); p.mask2n = c->nthroot - 1; p.lg = lg; p.n = c->N;
        auto post = [&](int e0, int m, u64* k) {
            p.e0 = e0; p.m = m; p.ks = k; p.ks_cs = (size_t)m * cs;
            ProfScope ps(LGPU_KCLASS_AUTOMORPHISM, st, 8.0 * N * nq * m * (s.odd ? 10 : 8), 1);
            expand_post_kernel<<<dim3((c->N + 255) / 256, (unsigned)nq, (unsigned)std::min(m, (int)kMaxGridZ)), 256, 0, st>>>(p);
            LGPU_CUDA_OK(cudaGetLastError());
            return 0;
        };
        auto pre = [&](int e0, int) -> const u64* { return X(i) + (size_t)e0 * ct; };
        if (keyswitch_chunks(c, level, s.cnt * B, *s.key, ks, st, pre, post)) return -1;
    }
    return 0;
}

// ---- Pack -----------------------------------------------------------------------------------------------------------
struct PackPlan {
    std::vector<int> step_i;          // tree level i of each step that has pairs
    std::vector<size_t> off;          // pairs of step s: pairs[off[s] .. off[s + 1])
    std::vector<Pair> pairs;
    std::vector<u64> galEl;
    std::vector<const GadgetCt*> key;
    int logStart = 0, logEnd = 0, nwork = 0, result = -1;
    int k0 = 0, nv = 0;               // the inputs the tree reads: positions k0 .. k0 + nv - 1 (0 <= idx < 2^inputLogGap, contiguous once sorted)
};

// getMinimumGap (:812-845) over the whole list (the reference stops scanning at a difference of 1; its keys come sorted from
// a map, here they are an argument and are all checked)
int minimum_gap(const int* idx, int n, long long& gap, int& log_gap) {
    gap = 0x7fffffffffffffffll;
    log_gap = 0;
    for (int i = 1; i < n; i++) {
        REQUIRE(idx[i - 1] <= idx[i], "getMinimumGap: invalid index list: element must be sorted from smallest to largest");
        REQUIRE(idx[i - 1] != idx[i], "getMinimumGap: invalid index list: contains duplicated elements");
        gap = std::min(gap, (long long)idx[i] - idx[i - 1]);
    }
    while ((gap & 1) == 0) { log_gap++; gap >>= 1; }
    return 0;
}

int pack_plan(const Ctx* c, const int* idx, int n_cts, int input_log_gap, bool zero_garbage, PackPlan& pl) {
    const int logN = c->logN;
    long long gap;
    int log_gap;
    if (n_cts > 1) {
        if (minimum_gap(idx, n_cts, gap, log_gap)) return -1;
    } else {
        gap = c->N; log_gap = logN;
    }
    pl.logStart = logN - input_log_gap;
    pl.logEnd = logN;
    if (!zero_garbage && gap > 0) pl.logEnd -= log_gap;
    REQUIRE(pl.logStart < pl.logEnd, "gaps between ciphertexts is smaller than inputLogGap > N");
    std::vector<int> loc((size_t)1 << input_log_gap, -1);    // map slot -> position (inputs - k0 at the first step, work slots after)
    pl.k0 = 0;
    while (pl.k0 < n_cts && idx[pl.k0] < 0) pl.k0++;
    for (int k = pl.k0; k < n_cts && idx[k] < (int)loc.size(); k++) loc[idx[k]] = pl.nv++;
    pl.off.push_back(0);
    for (int i = pl.logStart; i < pl.logEnd; i++) {
        const int t = 1 << (logN - 1 - i);
        const bool first = i == pl.logStart;
        const size_t before = pl.pairs.size();
        for (int jx = 0; jx < t; jx++) {
            const int a = loc[jx], b = loc[jx + t];
            if (a < 0 && b < 0) continue;
            Pair p;
            p.a = a; p.b = b;
            p.kind = a >= 0 && b >= 0 ? PAIR_AB : a >= 0 ? PAIR_A : PAIR_B;
            p.dst = first ? pl.nwork++ : (a >= 0 ? a : b);
            pl.pairs.push_back(p);
            loc[jx] = p.dst;
            loc[jx + t] = -1;
        }
        if (pl.pairs.size() == before) continue;
        pl.step_i.push_back(i);
        pl.off.push_back(pl.pairs.size());
        pl.galEl.push_back(i == 0 ? c->nthroot - 1 : galois_element(c, 1ll << (i - 1)));
    }
    pl.result = loc[0];
    REQUIRE(pl.result >= 0 && !pl.step_i.empty(),
            "Pack: no input ciphertext reaches slot 0 (the reference returns a nil ciphertext with a nil error)");
    return 0;
}

int pack_run(const Ctx* c, int level, const u64* cts_in, bool is_ntt, int n_cts, PackPlan& pl, u64* ct_out, int B, cudaStream_t st) {
    const size_t N = c->N, nq = level + 1, cs = nq * N, ct = 2 * cs;
    const int ch = batch_chunk();
    size_t max_pairs = 0;
    for (size_t s = 0; s + 1 < pl.off.size(); s++) max_pairs = std::max(max_pairs, pl.off[s + 1] - pl.off[s]);
    // the staging t and the key-switch outputs hold one chunk; the work block holds one ciphertext per pair of the first step
    const size_t work_cts = (size_t)pl.nwork * B, t_cts = std::min((size_t)ch, max_pairs * B), ks_cts = t_cts;
    const size_t ntt_cts = is_ntt ? 0 : (size_t)pl.nv * B;
    const size_t pair_words = (pl.pairs.size() * sizeof(Pair) + 7) / 8;
    Scratch buf;
    if (buf.alloc((work_cts + t_cts + ks_cts + ntt_cts) * ct + pair_words, st)) return -1;
    u64* work = buf.p;
    u64* t = work + work_cts * ct;
    u64* ks = t + t_cts * ct;
    u64* nttin = ks + ks_cts * ct;
    Pair* d_pairs = reinterpret_cast<Pair*>(nttin + ntt_cts * ct);
    LGPU_CUDA_OK(cudaMemcpyAsync(d_pairs, pl.pairs.data(), pl.pairs.size() * sizeof(Pair), cudaMemcpyHostToDevice, st));
    // the first step reads the inputs the tree uses, in place for an NTT-domain input, else their NTT (only those are transformed)
    const u64* src = cts_in + (size_t)pl.k0 * ct;
    size_t src_bs = (size_t)n_cts * ct;
    if (!is_ntt) {
        const RowMap rm = rows_range(0, 0, (int)nq);
        if (pl.nv == n_cts) {
            if (launch_ntt(c, rm, CSpan{src, N, cs}, Span{nttin, N, cs}, 2 * n_cts * B, NTT_CANONICAL, st)) return -1;
        } else {
            for (int b = 0; b < B; b++)
                if (launch_ntt(c, rm, CSpan{src + (size_t)b * src_bs, N, cs}, Span{nttin + (size_t)b * pl.nv * ct, N, cs}, 2 * pl.nv, NTT_CANONICAL, st))
                    return -1;
        }
        src = nttin;
        src_bs = (size_t)pl.nv * ct;
    }
    const int lg = log2_nthroot_half(c);
    const int logN = c->logN;
    const int s_exp = pl.logEnd - pl.logStart;
    for (size_t s = 0; s + 1 < pl.off.size(); s++) {
        const int i = pl.step_i[s];
        const int np = (int)(pl.off[s + 1] - pl.off[s]);
        const Pair* dp = d_pairs + pl.off[s];
        const bool first = s == 0;
        PackPreParams pp;
        pp.limbs = c->d_limbs; pp.pairs = dp; pp.batch = B;
        pp.src = first ? src : work; pp.src_ss = first ? ct : (size_t)B * ct; pp.src_bs = first ? src_bs : ct;
        pp.work = work; pp.work_ss = (size_t)B * ct; pp.t = t; pp.cs = cs;
        pp.k = (u64)1 << (logN - 1 - i); pp.lg = lg; pp.mask2n = c->nthroot - 1; pp.n = c->N; pp.scale = first ? 1 : 0;
        for (int r = 0; r < (int)nq; r++) {
            const u64 q = c->Q[r];
            pp.sc[r] = h_invmod(h_powmod(2, (u64)s_exp, q), q);
            pp.sc_sh[r] = shoup(pp.sc[r], q);
        }
        // the pairs are independent (each reads and writes only its own slots), so the pre pass can run chunk by chunk
        auto pre = [&](int e0, int m) -> const u64* {
            pp.e0 = e0; pp.m = m;
            ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * N * nq * m * 8, 1);
            pack_pre_kernel<<<dim3((c->N + 255) / 256, (unsigned)nq, (unsigned)std::min(m, (int)kMaxGridZ)), 256, 0, st>>>(pp);
            const cudaError_t err = cudaGetLastError();
            if (err != cudaSuccess) { set_error(std::string("pack_pre_kernel: ") + cudaGetErrorString(err)); return nullptr; }
            return t;
        };
        PackPostParams p;
        p.limbs = c->d_limbs; p.pairs = dp; p.batch = B; p.t = t; p.work = work; p.work_ss = (size_t)B * ct; p.cs = cs;
        p.galEl = pl.galEl[s]; p.mask2n = c->nthroot - 1; p.lg = lg; p.n = c->N;
        auto post = [&](int e0, int m, u64* k) {
            p.e0 = e0; p.m = m; p.ks = k; p.ks_cs = (size_t)m * cs;
            ProfScope ps(LGPU_KCLASS_AUTOMORPHISM, st, 8.0 * N * nq * m * 8, 1);
            pack_post_kernel<<<dim3((c->N + 255) / 256, (unsigned)nq, (unsigned)std::min(m, (int)kMaxGridZ)), 256, 0, st>>>(p);
            LGPU_CUDA_OK(cudaGetLastError());
            return 0;
        };
        if (keyswitch_chunks(c, level, np * B, *pl.key[s], ks, st, pre, post)) return -1;
    }
    // the result's work slot holds the B ciphertexts contiguously, which is ct_out's layout
    LGPU_CUDA_OK(cudaMemcpyAsync(ct_out, work + (size_t)pl.result * B * ct, (size_t)B * ct * 8, cudaMemcpyDeviceToDevice, st));
    return 0;
}

}  // namespace
}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_ring_packing_expand(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int is_ntt, int log_gap, const lgpu_galois_keys* gks,
                             uint64_t* ct_out, int batch, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "method is only supported for ring.Type = ring.Standard (X^{-2^{i}} does not exist in the sub-ring Z[X + X^{-1}])");
    REQUIRE(log_gap >= 0 && log_gap <= c.logN, "Expand: logGap out of range [0, LogN]");
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(is_ntt == 0 || is_ntt == 1, "is_ntt must be 0 or 1");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    const size_t ctb = (size_t)2 * (level + 1) * c.N * 8;
    REQUIRE(!overlaps(ct_out, ctb * batch * (c.N >> log_gap), ct_in, ctb * batch), "ct_out overlaps ct_in");
    GaloisKeySet ks;
    if (to_galois_keys(gks, ks)) return -1;
    std::vector<ExpandStep> sched = expand_schedule(&c, log_gap);
    for (ExpandStep& s : sched)
        if (lookup(&c, ks, level, s.galEl, s.key)) return -1;
    REQUIRE_DEVICE(ctx);
    return expand_run(&c, level, (const u64*)ct_in, is_ntt != 0, log_gap, sched, (u64*)ct_out, batch, (cudaStream_t)stream);
}

int lgpu_ring_packing_pack(lgpu_ctx* ctx, int level, const uint64_t* cts_in, int is_ntt, const int* idx, int n_cts, int input_log_gap,
                           int zero_garbage_slots, const lgpu_galois_keys* gks, uint64_t* ct_out, int batch, void* stream) {
    REQUIRE(ctx, "null context");
    REQUIRE(n_cts > 0, "len(cts) = 0");
    REQUIRE(idx, "null index array");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "procedure is only supported for ring.Type = ring.Standard (X^{2^{i}} does not exist in the sub-ring Z[X + X^{-1}])");
    REQUIRE(input_log_gap >= 0 && input_log_gap <= c.logN, "Pack: inputLogGap out of range [0, LogN]");
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(is_ntt == 0 || is_ntt == 1, "is_ntt must be 0 or 1");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(cts_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(cts_in) && AL(ct_out));
    const size_t ctb = (size_t)2 * (level + 1) * c.N * 8;
    REQUIRE(!overlaps(ct_out, ctb * batch, cts_in, ctb * batch * n_cts), "ct_out overlaps cts_in");
    PackPlan pl;
    if (pack_plan(&c, idx, n_cts, input_log_gap, zero_garbage_slots != 0, pl)) return -1;
    GaloisKeySet ks;
    if (to_galois_keys(gks, ks)) return -1;
    for (u64 g : pl.galEl) {
        const GadgetCt* k = nullptr;
        if (lookup(&c, ks, level, g, k)) return -1;
        pl.key.push_back(k);
    }
    REQUIRE_DEVICE(ctx);
    return pack_run(&c, level, (const u64*)cts_in, is_ntt != 0, n_cts, pl, (u64*)ct_out, batch, (cudaStream_t)stream);
}

}  // extern "C"
