// K9: the k-mer sharing counts of rsem-for-ebseq-calculate-clustering-info (EBSeq/calcClusteringInfo.cpp:101-130).
//
// The reference builds one record per k-mer start of the whole transcriptome, sorts the records with a base-by-base
// comparator and walks the groups of equal k-mers: a start position of transcript t counts when its group holds another
// transcript (numerator < denominator, :126).  Here the same count comes from one open-addressing hash table over all
// k-mers, in O(positions) data-parallel steps:
//   pack    the bases (one byte per base from the host, in chunks through a staging buffer) become 2-bit codes, 16 per
//           32-bit word, plus a 1-bit-per-base N mask, 32 per word.  N is code 0 with its mask bit set, so two k-mers are
//           equal exactly when their codes and masks are.
//   insert  one thread per start position: hash the k-mer (funnel shifts over the packed words, O(k / 16) loads), probe
//           linearly from its slot.  A slot key is a fingerprint of the hash above the global position + 1 of the k-mer's
//           first inserted occurrence.  A fingerprint match is verified base by base against that position, so the
//           result is exact for every k.  The slot's owner word goes EMPTY -> tid + 1 by CAS; a different tid makes it
//           SHARED, which never changes again.  SHARED therefore means: at least two transcripts hold the k-mer.
//   count   one thread per start position finds its slot again and, when the owner is SHARED, adds 1 to its transcript's
//           count.  Neighbouring positions mostly belong to one transcript: each warp adds one sum per transcript.
// When the table for all positions does not fit the device-memory budget, the k-mers are split by hash bits into P
// passes over one table: every k-mer (and so every group of equal k-mers) falls in exactly one pass, so the integer
// counts add up to the same result.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace rsem_b200 {

namespace {

constexpr uint32_t kShared = 0xffffffffu;       // owner word of a k-mer held by two or more transcripts
constexpr int kDefaultFpBits = 24;
constexpr int kThreads = 256;
constexpr uint64_t kStageBases = 64ull << 20;   // host -> device staging chunk (a multiple of 32 bases)
constexpr uint64_t kPadWords = 4;               // words after the packed arrays: chunk reads run up to 2 words past a k-mer
constexpr uint64_t kMargin = 512ull << 20;      // device memory left free when the budget comes from cudaMemGetInfo
constexpr uint64_t kSlotBytes = 12;             // 8-byte key + 4-byte owner

struct KmerDev {
    const uint32_t* code;   // 2-bit codes, base j at bits 2 (j % 16) of word j / 16
    const uint32_t* mask;   // N mask, base j at bit j % 32 of word j / 32
    const uint64_t* off;    // n + 1 transcript offsets
    uint64_t n, L;
    int k;
    int fp_bits;
    uint32_t passes, pass;
    unsigned long long* keys;
    uint32_t* owner;
    uint64_t slots;
    unsigned long long* counts;
    int* overflow;
};

// one staging chunk of byte codes (0..3 ACGT, 4 N) -> code / mask words; `first` is a multiple of 32
__global__ void kmer_pack_kernel(const uint8_t* __restrict__ b, uint64_t first, uint64_t n, uint32_t* __restrict__ code,
                                 uint32_t* __restrict__ mask) {
    const uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;   // mask word of the chunk (32 bases)
    if (w * 32 >= n) return;
    uint32_t c[2] = {0, 0}, m = 0;
    for (int j = 0; j < 32; ++j) {
        const uint64_t i = w * 32 + j;
        const uint32_t v = i < n ? b[i] : 0u;
        if (v > 3) m |= 1u << j;
        else c[j >> 4] |= v << (2 * (j & 15));
    }
    code[first / 16 + 2 * w] = c[0];
    code[first / 16 + 2 * w + 1] = c[1];
    mask[first / 32 + w] = m;
}

__device__ __forceinline__ uint32_t code_at(const uint32_t* __restrict__ code, uint64_t q) {   // 16 bases from q
    const uint64_t i = q >> 4;
    return __funnelshift_r(__ldg(code + i), __ldg(code + i + 1), (uint32_t)(q & 15) * 2);
}

__device__ __forceinline__ uint32_t mask_at(const uint32_t* __restrict__ mask, uint64_t q) {   // 32 bases from q
    const uint64_t i = q >> 5;
    return __funnelshift_r(__ldg(mask + i), __ldg(mask + i + 1), (uint32_t)(q & 31));
}

__device__ __forceinline__ uint32_t low_bits(int n) { return n >= 32 ? 0xffffffffu : (1u << n) - 1u; }

__device__ __forceinline__ uint64_t fmix64(uint64_t h) {
    h ^= h >> 33;
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
    h *= 0xc4ceb9fe1a85ec53ull;
    h ^= h >> 33;
    return h;
}

// a function of the k bases only (not of their position)
__device__ uint64_t kmer_hash(const KmerDev& d, uint64_t p) {
    uint64_t h = 0x9e3779b97f4a7c15ull;
    for (int i = 0; i < d.k; i += 32) {
        const int rem = d.k - i;
        const uint32_t c0 = code_at(d.code, p + i) & low_bits(2 * min(rem, 16));
        const uint32_t c1 = rem > 16 ? code_at(d.code, p + i + 16) & low_bits(2 * (rem - 16)) : 0u;
        const uint32_t m = mask_at(d.mask, p + i) & low_bits(rem);
        h ^= (uint64_t)c0 | ((uint64_t)c1 << 32);
        h *= 0x9e3779b97f4a7c15ull;
        h ^= h >> 29;
        h ^= m;
        h *= 0xbf58476d1ce4e5b9ull;
        h ^= h >> 32;
    }
    return fmix64(h ^ (uint64_t)d.k);
}

__device__ bool kmer_equal(const KmerDev& d, uint64_t p, uint64_t q) {
    for (int i = 0; i < d.k; i += 16)
        if ((code_at(d.code, p + i) ^ code_at(d.code, q + i)) & low_bits(2 * min(d.k - i, 16))) return false;
    for (int i = 0; i < d.k; i += 32)
        if ((mask_at(d.mask, p + i) ^ mask_at(d.mask, q + i)) & low_bits(d.k - i)) return false;
    return true;
}

// last transcript t in [lo, hi] with off[t] <= g (empty transcripts share an offset with the next one)
__device__ __forceinline__ uint64_t find_transcript(const uint64_t* __restrict__ off, uint64_t lo, uint64_t hi, uint64_t g) {
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) / 2;
        if (__ldg(off + mid) <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Position g of this thread, its transcript t, and whether a k-mer starts there.  The CTA first locates the transcripts
// of its first and last position, so each thread searches only between those two (usually one or two transcripts).
__device__ __forceinline__ bool locate(const KmerDev& d, uint64_t& g, uint64_t& t) {
    __shared__ uint64_t range[2];
    const uint64_t first = blockIdx.x * (uint64_t)blockDim.x;
    if (threadIdx.x < 2) {
        const uint64_t at = threadIdx.x == 0 ? first : min(first + blockDim.x, d.L) - 1;
        range[threadIdx.x] = find_transcript(d.off, 0, d.n - 1, at);
    }
    __syncthreads();
    g = first + threadIdx.x;
    if (g >= d.L) return false;
    t = find_transcript(d.off, range[0], range[1], g);
    return g + (uint64_t)d.k <= __ldg(d.off + t + 1);
}

struct Probe {
    uint64_t slot;
    uint64_t key;        // fingerprint << pos_bits | (g + 1)
    uint64_t fp;
};

__device__ __forceinline__ Probe make_probe(const KmerDev& d, uint64_t h, uint64_t g) {
    const int pos_bits = 64 - d.fp_bits;
    Probe pr;
    pr.fp = h & ((1ull << d.fp_bits) - 1);   // the low bits; the pass takes the high 32, the slot a remix of all 64
    pr.key = (pr.fp << pos_bits) | (g + 1);
    pr.slot = __umul64hi(fmix64(h ^ 0x2545f4914f6cdd1dull), d.slots);
    return pr;
}

__device__ __forceinline__ uint32_t pass_of(const KmerDev& d, uint64_t h) {
    return (uint32_t)(((h >> 32) * (uint64_t)d.passes) >> 32);
}

// does the occupied key `cur` hold the k-mer starting at g?
__device__ __forceinline__ bool holds(const KmerDev& d, uint64_t cur, const Probe& pr, uint64_t g) {
    const int pos_bits = 64 - d.fp_bits;
    if ((cur >> pos_bits) != pr.fp) return false;
    const uint64_t q = (cur & ((1ull << pos_bits) - 1)) - 1;
    return q == g || kmer_equal(d, q, g);
}

__global__ void __launch_bounds__(kThreads) kmer_insert_kernel(KmerDev d) {
    uint64_t g, t;
    if (!locate(d, g, t)) return;
    const uint64_t h = kmer_hash(d, g);
    if (pass_of(d, h) != d.pass) return;
    const Probe pr = make_probe(d, h, g);
    uint64_t slot = pr.slot;
    for (uint64_t probes = 0;; ++probes) {
        if (probes == d.slots) { atomicExch(d.overflow, 1); return; }
        // a key goes from 0 to its final value once: a stale 0 only sends this thread to the CAS, which reads the truth
        uint64_t cur = __ldcg(d.keys + slot);
        if (cur == 0) {
            cur = atomicCAS(d.keys + slot, 0ull, (unsigned long long)pr.key);
            if (cur == 0) break;   // this position is the k-mer's first occurrence in the table
        }
        if (holds(d, cur, pr, g)) break;
        if (++slot == d.slots) slot = 0;
    }
    // EMPTY -> tid + 1 -> SHARED; an owner read as another tid is current (tids are written once, before SHARED)
    const uint32_t me = (uint32_t)t + 1;
    uint32_t o = __ldcg(d.owner + slot);
    if (o == 0) o = atomicCAS(d.owner + slot, 0u, me);
    if (o != 0 && o != me && o != kShared) atomicExch(d.owner + slot, kShared);
}

__global__ void __launch_bounds__(kThreads) kmer_count_kernel(KmerDev d) {
    uint64_t g = 0, t = 0;
    bool valid = locate(d, g, t);
    bool shared = false;
    if (valid) {
        const uint64_t h = kmer_hash(d, g);
        valid = pass_of(d, h) == d.pass;
        if (valid) {
            const Probe pr = make_probe(d, h, g);
            uint64_t slot = pr.slot;
            for (uint64_t probes = 0;; ++probes) {
                const uint64_t cur = d.keys[slot];
                if (cur == 0 || probes == d.slots) { atomicExch(d.overflow, 1); valid = false; break; }   // not inserted
                if (holds(d, cur, pr, g)) { shared = d.owner[slot] == kShared; break; }
                if (++slot == d.slots) slot = 0;
            }
        }
    }
    // one atomic per transcript of the warp
    const unsigned same = __match_any_sync(0xffffffffu, valid ? t : ~0ull);
    const unsigned hits = __ballot_sync(0xffffffffu, shared) & same;
    if (valid && hits && (threadIdx.x & 31) == (unsigned)(__ffs(same) - 1)) atomicAdd(d.counts + t, (unsigned long long)__popc(hits));
}

struct Buffers {   // device memory and events of one call, released on every return path
    std::vector<void*> mem;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaStream_t st = nullptr;
    ~Buffers() {
        if (st) cudaStreamSynchronize(st);
        for (void* p : mem) cudaFree(p);
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
    template <class T>
    cudaError_t alloc(T** p, size_t bytes) {
        cudaError_t e = cudaMalloc((void**)p, std::max<size_t>(bytes, 16));
        if (e == cudaSuccess) mem.push_back((void*)*p);
        return e;
    }
    void release(void* p) {
        auto it = std::find(mem.begin(), mem.end(), p);
        if (it != mem.end()) { cudaFree(p); mem.erase(it); }
    }
};

float elapsed(cudaEvent_t a, cudaEvent_t b) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}

}  // namespace

int kmer_shared(rsem_b200_ctx* ctx, const rsem_b200_kmer_params* p, uint64_t* counts, rsem_b200_kmer_stats* stats) {
    const uint64_t n = p->n_transcripts, L = p->offsets[n];
    const int k = p->k, fp_bits = p->fingerprint_bits ? p->fingerprint_bits : kDefaultFpBits;
    uint64_t positions = 0;
    for (uint64_t t = 0; t < n; ++t) {
        const uint64_t len = p->offsets[t + 1] - p->offsets[t];
        if (len >= (uint64_t)k) positions += len - k + 1;
    }
    RB_ARG(L + 1 < (1ull << (64 - fp_bits)), "kmer_shared: too many bases for the slot key's position field");
    std::fill(counts, counts + n, 0);
    rsem_b200_kmer_stats s{};
    s.positions = positions;
    if (positions == 0) {
        if (stats) *stats = s;
        return 0;
    }

    Buffers B;
    B.st = ctx->stream;
    const cudaStream_t st = ctx->stream;
    for (auto& e : B.ev) RB_CUDA(cudaEventCreate(&e));
    KmerDev d{};
    d.n = n;
    d.L = L;
    d.k = k;
    d.fp_bits = fp_bits;
    const uint64_t n_code = L / 16 + kPadWords, n_mask = L / 32 + kPadWords;
    s.input_bytes = 4 * (n_code + n_mask) + 8 * (n + 1) + 8 * n + sizeof(int);
    uint32_t *code = nullptr, *mask = nullptr;
    uint64_t* off = nullptr;
    RB_CUDA(B.alloc(&code, 4 * n_code));
    RB_CUDA(B.alloc(&mask, 4 * n_mask));
    RB_CUDA(B.alloc(&off, 8 * (n + 1)));
    RB_CUDA(B.alloc(&d.counts, 8 * n));
    RB_CUDA(B.alloc(&d.overflow, sizeof(int)));

    // pack through one staging buffer
    RB_CUDA(cudaEventRecord(B.ev[0], st));
    RB_CUDA(cudaMemsetAsync(code, 0, 4 * n_code, st));
    RB_CUDA(cudaMemsetAsync(mask, 0, 4 * n_mask, st));
    RB_CUDA(cudaMemcpyAsync(off, p->offsets, 8 * (n + 1), cudaMemcpyHostToDevice, st));
    RB_CUDA(cudaMemsetAsync(d.counts, 0, 8 * n, st));
    RB_CUDA(cudaMemsetAsync(d.overflow, 0, sizeof(int), st));
    {
        uint8_t* stage = nullptr;
        const uint64_t chunk = std::min<uint64_t>(kStageBases, (L + 31) / 32 * 32);
        RB_CUDA(B.alloc(&stage, chunk));
        for (uint64_t first = 0; first < L; first += chunk) {
            const uint64_t len = std::min(chunk, L - first);
            // stream order keeps the next copy into `stage` behind the kernel that reads it
            RB_CUDA(cudaMemcpyAsync(stage, p->bases + first, len, cudaMemcpyHostToDevice, st));
            const uint64_t words = (len + 31) / 32;
            kmer_pack_kernel<<<(unsigned)((words + kThreads - 1) / kThreads), kThreads, 0, st>>>(stage, first, len, code, mask);
            RB_CUDA(cudaGetLastError());
            ctx->launches++;
        }
        RB_CUDA(cudaEventRecord(B.ev[1], st));
        RB_CUDA(cudaStreamSynchronize(st));
        B.release(stage);
        s.pack_ms = elapsed(B.ev[0], B.ev[1]);
    }
    d.code = code;
    d.mask = mask;
    d.off = off;

    // table size and passes: at most half the slots filled in a pass (the distinct k-mers of a pass never outnumber its
    // positions, about positions / P)
    uint64_t budget = p->max_device_bytes;
    if (budget == 0) {
        size_t free_b = 0, total_b = 0;
        RB_CUDA(cudaMemGetInfo(&free_b, &total_b));
        budget = free_b > kMargin ? s.input_bytes + (free_b - kMargin) : 0;
    }
    const uint64_t slots_max = budget > s.input_bytes ? (budget - s.input_bytes) / kSlotBytes : 0;
    RB_ARG(slots_max >= 1024, "kmer_shared: the device-memory budget leaves no room for a hash table");
    const uint64_t passes = (2 * positions + slots_max - 1) / slots_max;
    RB_ARG(passes <= 65536, "kmer_shared: the device-memory budget needs more than 65536 passes");
    d.passes = (uint32_t)passes;
    d.slots = std::min(slots_max, 2 * ((positions + passes - 1) / passes) + 64);
    RB_CUDA(B.alloc(&d.keys, 8 * d.slots));
    RB_CUDA(B.alloc(&d.owner, 4 * d.slots));
    s.passes = (int32_t)passes;
    s.table_slots = d.slots;
    s.table_bytes = kSlotBytes * d.slots;

    const unsigned grid = (unsigned)((L + kThreads - 1) / kThreads);
    double insert_ms = 0, count_ms = 0;
    for (uint32_t pass = 0; pass < d.passes; ++pass) {
        d.pass = pass;
        RB_CUDA(cudaEventRecord(B.ev[1], st));   // the table's clearing counts as insert time
        RB_CUDA(cudaMemsetAsync(d.keys, 0, 8 * d.slots, st));
        RB_CUDA(cudaMemsetAsync(d.owner, 0, 4 * d.slots, st));
        kmer_insert_kernel<<<grid, kThreads, 0, st>>>(d);
        RB_CUDA(cudaGetLastError());
        RB_CUDA(cudaEventRecord(B.ev[2], st));
        kmer_count_kernel<<<grid, kThreads, 0, st>>>(d);
        RB_CUDA(cudaGetLastError());
        RB_CUDA(cudaEventRecord(B.ev[3], st));
        ctx->launches += 2;
        RB_CUDA(cudaEventSynchronize(B.ev[3]));
        insert_ms += elapsed(B.ev[1], B.ev[2]);
        count_ms += elapsed(B.ev[2], B.ev[3]);
    }
    int overflow = 0;
    RB_CUDA(cudaMemcpyAsync(&overflow, d.overflow, sizeof(int), cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaMemcpyAsync(counts, d.counts, 8 * n, cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
    if (overflow) {
        set_error("kmer_shared: the hash table overflowed");
        return RSEM_B200_ERR_CUDA;
    }
    s.insert_ms = insert_ms;
    s.count_ms = count_ms;
    if (stats) *stats = s;
    return 0;
}

}  // namespace rsem_b200
