// MT19937 jump-ahead on the host (Haramoto, Matsumoto, Nishimura, Panneton, L'Ecuyer 2008, "Efficient jump ahead for
// F2-linear random number generators").
//
// The untempered words y_n of the generator satisfy one linear recurrence over GF(2) for n >= 1: its characteristic
// polynomial p(x), of degree 19937.  For a window S of 624 consecutive words of the sequence (all past the seed's first
// word) and the shift-by-one map T, T^J S = g(T) S with g(x) = x^J mod p(x).  p is found once per process by
// Berlekamp-Massey over 2 * 19937 output bits; x^J mod p by square-and-multiply on 19937-bit polynomials in 64-bit
// words (a square in GF(2)[x] is the carry-less product of a polynomial with itself: its bits spread apart).
//
// A jump moves the state's array by whole blocks of 624 words (one boost twist each) and sets its index, so that the
// result is exactly the state boost::mt19937 reaches after J draws.  g(T) S is evaluated by Horner's rule over the 32
// blocks of 624 coefficients: acc = twist(acc) ^ C_b, where C_b[j] = sum_i g_{624 b + i} s_{i + j} over the 1248 words
// s that follow S.  sim_kernels.cu applies the same scheme on the device.
#include <cstring>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace rsem_b200 {

namespace {

constexpr int kN = 624, kM = 397, kDeg = 19937;
constexpr int kWords = kMtPolyWords;  // 312 x 64 = 19968 >= 19937 + 1 bits

uint32_t twist_word(uint32_t a, uint32_t b, uint32_t c) {
    const uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return c ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

// boost's twist of the whole array, in place (the four dependent ranges in order)
void twist(uint32_t* x) {
    for (int i = 0; i < kN; ++i) x[i] = twist_word(x[i], x[(i + 1) % kN], x[(i + kM) % kN]);
}

uint32_t temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    return y ^ (y >> 18);
}

bool bit(const std::vector<uint64_t>& a, size_t i) { return (a[i >> 6] >> (i & 63)) & 1; }

// p(x): Berlekamp-Massey on bit 0 of 2 * 19937 outputs.  The minimal polynomial of any nonzero output bit sequence is
// the characteristic polynomial, which is irreducible for MT19937.
std::vector<uint64_t> charpoly() {
    const int n_bits = 2 * kDeg;
    const int nw = (n_bits + 63) / 64 + 2;
    std::vector<uint64_t> r(nw, 0);  // r[k] = s_{n_bits - 1 - k}: the discrepancy reads a contiguous run of it
    uint32_t x[kN];
    x[0] = 5489u;
    for (int i = 1; i < kN; ++i) x[i] = 1812433253u * (x[i - 1] ^ (x[i - 1] >> 30)) + (uint32_t)i;
    for (int n = 0; n < n_bits; ++n) {
        if (n % kN == 0) twist(x);
        const size_t k = (size_t)(n_bits - 1 - n);
        if (temper(x[n % kN]) & 1u) r[k >> 6] |= 1ull << (k & 63);
    }
    const int cw = kWords + 2;
    std::vector<uint64_t> C(2 * cw, 0), B(2 * cw, 0), T;
    C[0] = B[0] = 1;
    int L = 0, m = 1;
    for (int n = 0; n < n_bits; ++n) {
        // d = sum_{i=0..L} C_i s_{n-i} = parity(C & r[off ..]), off = n_bits - 1 - n
        const size_t off = (size_t)(n_bits - 1 - n);
        const size_t q = off >> 6, sh = off & 63;
        uint64_t acc = 0;
        for (int j = 0; j <= L / 64; ++j) {
            uint64_t w = r[q + j] >> sh;
            if (sh) w |= r[q + j + 1] << (64 - sh);
            acc ^= C[j] & w;
        }
        if (!__builtin_parityll(acc)) { ++m; continue; }
        const bool grow = 2 * L <= n;
        if (grow) T = C;
        const int qw = m >> 6, bs = m & 63;
        for (int j = cw - 1; j >= 0; --j) {
            uint64_t w = B[j] << bs;
            if (bs && j) w |= B[j - 1] >> (64 - bs);
            if (j + qw < 2 * cw) C[j + qw] ^= w;
        }
        if (grow) { L = n + 1 - L; B = T; m = 1; }
        else ++m;
    }
    std::vector<uint64_t> p(kWords, 0);
    if (L != kDeg) return {};
    for (int k = 0; k <= kDeg; ++k)  // p_k = C_{L - k}
        if (bit(C, (size_t)(kDeg - k))) p[k >> 6] |= 1ull << (k & 63);
    return p;
}

// p shifted left by 0..63 bits, 313 words each
const std::vector<uint64_t>& shifted_p() {
    static std::once_flag once;
    static std::vector<uint64_t> sp;
    std::call_once(once, []() {
        const std::vector<uint64_t> p = charpoly();
        if (p.empty()) return;
        sp.assign(64 * (kWords + 1), 0);
        for (int s = 0; s < 64; ++s)
            for (int j = 0; j <= kWords; ++j) {
                uint64_t w = j < kWords ? p[j] << s : 0;
                if (s && j) w |= p[j - 1] >> (64 - s);
                sp[(size_t)s * (kWords + 1) + j] = w;
            }
    });
    return sp;
}

// a (2 * kWords words, degree < 2 * 19937) mod p, in place
void reduce(std::vector<uint64_t>& a, const std::vector<uint64_t>& sp) {
    for (int i = 2 * kDeg - 2; i >= kDeg; --i) {
        if (!((a[i >> 6] >> (i & 63)) & 1)) continue;
        const int sft = i - kDeg;
        const uint64_t* ps = &sp[(size_t)(sft & 63) * (kWords + 1)];
        uint64_t* dst = &a[sft >> 6];
        for (int j = 0; j <= kWords; ++j) dst[j] ^= ps[j];
    }
}

uint64_t spread(uint32_t v) {  // bit i -> bit 2i
    uint64_t x = v;
    x = (x | (x << 16)) & 0x0000ffff0000ffffull;
    x = (x | (x << 8)) & 0x00ff00ff00ff00ffull;
    x = (x | (x << 4)) & 0x0f0f0f0f0f0f0f0full;
    x = (x | (x << 2)) & 0x3333333333333333ull;
    x = (x | (x << 1)) & 0x5555555555555555ull;
    return x;
}

}  // namespace

bool mt_jump_poly(uint64_t J, uint64_t out[kMtPolyWords]) {
    const std::vector<uint64_t>& sp = shifted_p();
    if (sp.empty()) return false;
    std::vector<uint64_t> a(2 * kWords + 2, 0), sq(2 * kWords + 2, 0);
    a[0] = 1;
    for (int b = 63; b >= 0; --b) {
        std::fill(sq.begin(), sq.end(), 0);
        for (int j = 0; j < kWords; ++j) {  // carry-less square
            sq[2 * j] = spread((uint32_t)a[j]);
            sq[2 * j + 1] = spread((uint32_t)(a[j] >> 32));
        }
        reduce(sq, sp);
        a.swap(sq);
        if ((J >> b) & 1) {  // times x
            for (int j = kWords; j > 0; --j) a[j] = (a[j] << 1) | (a[j - 1] >> 63);
            a[0] <<= 1;
            if ((a[kDeg >> 6] >> (kDeg & 63)) & 1)
                for (int j = 0; j < kWords; ++j) a[j] ^= sp[j];
        }
    }
    std::memcpy(out, a.data(), kMtPolyWords * sizeof(uint64_t));
    return true;
}

MtJumpPlan mt_jump_plan(uint32_t idx, uint64_t J) {
    if (J == 0) return {idx, 0};
    const uint64_t t = idx + J;
    if (t <= (uint64_t)kN) return {(uint32_t)t, 0};
    const uint64_t k = (t - 1) / kN;
    return {(uint32_t)(t - k * kN), k};
}

int mt_jump_blocks(const uint64_t poly[kMtPolyWords], uint32_t blocks[kMtJumpBlocks * kMtBlockWords]) {
    std::memset(blocks, 0, kMtJumpBlocks * kMtBlockWords * sizeof(uint32_t));
    int nb = 0;
    for (int i = 0; i < kDeg; ++i)
        if ((poly[i >> 6] >> (i & 63)) & 1) {
            const int b = i / kN, o = i % kN;
            blocks[b * kMtBlockWords + (o >> 5)] |= 1u << (o & 31);
            nb = b + 1;
        }
    return nb;
}

}  // namespace rsem_b200

using namespace rsem_b200;

extern "C" int rsem_b200_mt19937_jump(const uint32_t state_in[625], uint64_t J, uint32_t state_out[625]) {
    RB_ARG(state_in && state_out, "NULL argument");
    RB_ARG(state_in[kN] <= (uint32_t)kN, "state index above 624");
    const MtJumpPlan plan = mt_jump_plan(state_in[kN], J);
    std::vector<uint32_t> s(2 * kN);
    std::memcpy(s.data(), state_in, kN * sizeof(uint32_t));
    if (plan.blocks) {
        // S = the array one block on (exact from any state), then Horner over the blocks of x^(624 (blocks - 1)) mod p
        twist(s.data());
        std::memcpy(s.data() + kN, s.data(), kN * sizeof(uint32_t));
        twist(s.data() + kN);
        std::vector<uint64_t> poly(kMtPolyWords);
        RB_ARG(mt_jump_poly((plan.blocks - 1) * kN, poly.data()), "mt19937 characteristic polynomial not found");
        std::vector<uint32_t> h(kMtJumpBlocks * kMtBlockWords);
        const int nb = mt_jump_blocks(poly.data(), h.data());
        std::vector<uint32_t> acc(kN, 0);
        for (int b = nb - 1; b >= 0; --b) {
            twist(acc.data());
            const uint32_t* hb = &h[(size_t)b * kMtBlockWords];
            for (int i = 0; i < kN; ++i)
                if ((hb[i >> 5] >> (i & 31)) & 1)
                    for (int j = 0; j < kN; ++j) acc[j] ^= s[i + j];
        }
        std::memcpy(s.data(), acc.data(), kN * sizeof(uint32_t));
    }
    std::memcpy(state_out, s.data(), kN * sizeof(uint32_t));
    state_out[kN] = plan.idx;
    return 0;
}
