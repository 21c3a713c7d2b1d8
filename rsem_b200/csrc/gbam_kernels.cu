// K10: the per-alignment work of rsem-tbam2gbam (BamConverter.h:92-303, bc_aux.h, tr2chr in sam_utils.h:137-208).
//
// The reference converts one alignment at a time on one thread and collapses the alignments of a read in a std::map
// keyed by (tid, pos, strand, CIGAR).  Here one batch of whole groups (runs of one read name) goes through:
//   sizes    one thread per unit (a record or a mate pair): the converted size of each record (tr2chr's CIGAR length,
//            one XS removed, XS:A appended when the CIGAR has an N); exclusive scan -> offsets in the scratch buffer
//   convert  the same walk, writing: tid / pos / bin / flags / isize, the new CIGAR, the complement-reversed sequence,
//            the reversed qualities, MD rewritten on '-' transcripts, XS handled; mates get each other's new pos;
//            per unit: its ZW as float (bam_aux2f) and where mate 1's and mate 2's ZW values now lie
//   sort     one stable merge sort of unit indices by (group, key of mate 1, key of mate 2); the comparator reads the
//            converted records.  Stable: a run of equal keys keeps its units in input order
//   collapse one thread per sorted position marks run heads; one thread per head sums the run's ZW in float in input
//            order (the reference's `+=`), looks MAPQ up in the host-built threshold table, and sizes the output
//   emit     exclusive scan of the sizes; one thread per head writes block_size + record (the first unit of the run, with
//            ZW and MAPQ patched), or the input bytes of an unmapped unit
#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace rsem_b200 {

struct GbamState {
    const rsem_b200_gbam_tables* tables_key = nullptr;
    int32_t* out_tid = nullptr;
    uint8_t* minus = nullptr;
    int32_t* length = nullptr;
    int64_t* exon_off = nullptr;
    int32_t* exon_start = nullptr;
    int32_t* exon_end = nullptr;
    float* mapq_prb = nullptr;
    // batch scratch, grown as needed
    uint8_t *data = nullptr, *conv = nullptr, *out = nullptr, *head = nullptr;
    uint64_t *rec_off = nullptr, *conv_off = nullptr, *out_off = nullptr;
    uint32_t *unit_rec = nullptr, *unit_group = nullptr, *keys = nullptr;
    int32_t *unit_tr = nullptr, *zw = nullptr;    // zw: 2 per unit, offsets of the ZW values from the unit's first byte
    float *prb = nullptr, *run_prb = nullptr;
    void* temp = nullptr;
    unsigned long long* err = nullptr;
    size_t sz_data = 0, sz_conv = 0, sz_out = 0, sz_rec = 0, sz_unit = 0, sz_temp = 0;
    cudaEvent_t ev[2] = {nullptr, nullptr};
};

namespace {

constexpr int kThreads = 256;
enum Bad : unsigned { kBadBase = 1, kBadPos, kBadExon, kBadChr, kBadMateZw, kBadPrb, kBadAux };

struct Tables {
    const int32_t* out_tid;
    const uint8_t* minus;
    const int32_t* length;
    const int64_t* exon_off;
    const int32_t* exon_start;
    const int32_t* exon_end;
    const float* mapq_prb;
};

struct Batch {
    const uint8_t* data;
    const uint64_t* rec_off;
    const uint32_t* unit_rec;
    const uint32_t* unit_group;
    const int32_t* unit_tr;
    uint32_t n_units;
};

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }
__device__ __forceinline__ void wr32(uint8_t* p, uint32_t v) { p[0] = v & 255; p[1] = (v >> 8) & 255; p[2] = (v >> 16) & 255; p[3] = v >> 24; }
__device__ __forceinline__ void wr16(uint8_t* p, uint16_t v) { p[0] = v & 255; p[1] = v >> 8; }

__device__ __forceinline__ void flag_bad(unsigned long long* err, uint32_t unit, unsigned why) {
    atomicMin(err, ((unsigned long long)unit << 8) | why);
}

// tr2chr (sam_utils.h:137-208), literally: the linear walk over the exons.  cig: where the CIGAR words go (unaligned),
// nullptr to count only.  Returns the number of CIGAR operations, or -1 when the walk runs off the exons (the
// reference's assert(i < s)).
__device__ int tr2chr(const Tables& T, int t, int sp, int ep, int& pos, uint8_t* cig, bool& has_n) {
    const int length = T.length[t];
    const int32_t* st = T.exon_start + T.exon_off[t];
    const int32_t* en = T.exon_end + T.exon_off[t];
    const int s = (int)(T.exon_off[t + 1] - T.exon_off[t]);
    int n = 0;
    has_n = false;
    auto put = [&](uint32_t op) { if (cig) wr32(cig + 4 * n, op); ++n; };
    if (T.minus[t]) {
        const int tmp = sp;
        sp = length - ep + 1;
        ep = length - tmp + 1;
    }
    if (s == 0) return -1;
    if (ep < 1 || sp > length) {   // entirely in the poly(A) tail
        pos = sp > length ? en[s - 1] : st[0] - 1;
        put((uint32_t)(ep - sp + 1) << 4 | 1u);
        return n;
    }
    if (sp < 1) {
        put((uint32_t)(1 - sp) << 4 | 1u);
        sp = 1;
    }
    int i, oldlen = 0, curlen = 0;
    for (i = 0; i < s; i++) {
        oldlen = curlen;
        curlen += en[i] - st[i] + 1;
        if (curlen >= sp) break;
    }
    if (i >= s) return -1;
    pos = st[i] + (sp - oldlen - 1) - 1;
    while (curlen < ep && i < s) {
        put((uint32_t)(curlen - sp + 1) << 4 | 0u);
        ++i;
        if (i >= s) continue;
        put((uint32_t)(st[i] - en[i - 1] - 1) << 4 | 3u);
        has_n = true;
        oldlen = curlen;
        sp = oldlen + 1;
        curlen += en[i] - st[i] + 1;
    }
    if (i >= s) put((uint32_t)(ep - length) << 4 | 1u);
    else put((uint32_t)(ep - sp + 1) << 4 | 0u);
    return n;
}

// SAM spec 5.3 / hts_reg2bin(beg, end, 14, 5) of htslib 1.3 (hts.h:578-584)
__device__ int reg2bin(int64_t beg, int64_t end) {
    --end;
    if (beg >> 14 == end >> 14) return (int)(((1 << 15) - 1) / 7 + (beg >> 14));
    if (beg >> 17 == end >> 17) return (int)(((1 << 12) - 1) / 7 + (beg >> 17));
    if (beg >> 20 == end >> 20) return (int)(((1 << 9) - 1) / 7 + (beg >> 20));
    if (beg >> 23 == end >> 23) return (int)(((1 << 6) - 1) / 7 + (beg >> 23));
    if (beg >> 26 == end >> 26) return (int)(((1 << 3) - 1) / 7 + (beg >> 26));
    return 0;
}

__device__ __forceinline__ uint8_t md_opp(uint8_t c) {   // getOpp on A/C/G/T only (BamConverter.h:270)
    switch (c) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A'; }
    return c;
}

// modifyTags' MD rewrite (BamConverter.h:251-290), literally: runs of digits keep their order, runs of other letters
// are reversed and complemented, a run starting with '^' keeps the '^' in front; every run moves to its mirrored place
__device__ void md_flip(const uint8_t* mis, uint8_t* tmp, int len) {
    int cur_type = -1, fr = -1;
    for (int i = 0; i <= len; i++) {
        const int type = i < len ? (mis[i] >= '0' && mis[i] <= '9') : -2;
        if (cur_type != type) {
            if (cur_type == 0) {
                int base = len - 1, f = fr;
                if (mis[f] == '^') { tmp[len - i] = mis[f]; ++f; ++base; }
                for (int j = f; j < i; j++) tmp[base - j] = md_opp(mis[j]);
            } else if (cur_type == 1) {
                const int base = len - i - fr;
                for (int j = fr; j < i; j++) tmp[base + j] = mis[j];
            }
            cur_type = type;
            fr = i;
        }
    }
}

struct Conv {          // one converted record: its size, and (write pass) where ZW went
    uint32_t bytes;    // block_size + 4
    int32_t zw;        // offset of the ZW field's type byte from the record's block_size, -1 if none
    int32_t pos;
    float prb;         // bam_aux2f of the first ZW, 1.0 without one
    unsigned bad;
};

// convert() + modifyTags() of one record (BamConverter.h:150-191, 251-303).  in: the record after its block_size.
// o: where block_size goes, or nullptr (sizes pass).
__device__ Conv convert(const Tables& T, int t, const uint8_t* in, uint32_t in_size, uint8_t* o) {
    Conv r{0, -1, 0, 1.0f, 0};
    const int32_t pos = (int32_t)rd32(in + 4);
    const uint32_t l_qname = in[8];
    const uint32_t n_cig = rd16(in + 12);
    uint16_t flag = rd16(in + 14);
    const int32_t l_seq = (int32_t)rd32(in + 16);
    const bool minus = T.minus[t] != 0, paired = flag & 1;
    const int32_t tid = T.out_tid[t];
    if (tid < 0) { r.bad = kBadChr; return r; }
    const uint8_t* seq = in + 32 + l_qname + 4 * n_cig;
    const uint8_t* qual = seq + (l_seq + 1) / 2;
    const uint8_t* aux = qual + l_seq;
    const uint8_t* aux_end = in + in_size;
    int new_pos = 0;
    bool has_n = false;
    const int nc = tr2chr(T, t, pos + 1, pos + l_seq, new_pos, nullptr, has_n);
    if (nc < 0) { r.bad = kBadExon; return r; }
    if (new_pos < 0) { r.bad = kBadPos; return r; }
    r.pos = new_pos;
    // optional fields: the first XS goes, XS:A:<strand> is appended when the CIGAR has an N
    const uint8_t* xs = nullptr;
    const uint8_t* md = nullptr;
    const uint8_t* zw = nullptr;
    uint32_t xs_len = 0;
    // every byte of the optional block must belong to a field: stray bytes at its end are refused here, so that the
    // write pass below, which copies field by field, writes exactly l_aux bytes
    for (const uint8_t* a = aux; a < aux_end;) {
        if (a + 3 > aux_end) { r.bad = kBadAux; return r; }
        const int len = aux_len(a + 2, aux_end);
        if (len == 0 || a + 2 + len > aux_end) { r.bad = kBadAux; return r; }
        if (a[0] == 'X' && a[1] == 'S' && !xs) { xs = a; xs_len = 2 + len; }
        if (a[0] == 'M' && a[1] == 'D' && !md) md = a;
        if (a[0] == 'Z' && a[1] == 'W' && !zw) zw = a;
        a += 2 + len;
    }
    const uint32_t l_aux = (uint32_t)(aux_end - aux) - xs_len + (has_n ? 4 : 0);
    const uint32_t block = 32 + l_qname + 4 * (uint32_t)nc + (uint32_t)(l_seq + 1) / 2 + (uint32_t)l_seq + l_aux;
    r.bytes = 4 + block;
    if (zw) {   // bam_aux2f: 'd' or 'f', anything else reads as 0
        if (zw[2] == 'f') r.prb = __uint_as_float(rd32(zw + 3));
        else if (zw[2] == 'd') r.prb = (float)__longlong_as_double((long long)((uint64_t)rd32(zw + 3) | (uint64_t)rd32(zw + 7) << 32));
        else r.prb = 0.0f;
    }
    if (!o) return r;

    // core
    uint8_t* w = o + 4;
    wr32(o, block);
    wr32(w, (uint32_t)tid);
    wr32(w + 4, (uint32_t)new_pos);
    if (minus) {
        flag ^= 16;
        if (paired) flag ^= 32;
    }
    wr32(w + 16, (uint32_t)l_seq);
    wr32(w + 20, paired ? (uint32_t)tid : rd32(in + 20));
    wr32(w + 24, rd32(in + 24));
    const int32_t isize = (int32_t)rd32(in + 28);
    wr32(w + 28, (uint32_t)(minus && paired ? -isize : isize));
    for (uint32_t k = 0; k < l_qname; ++k) w[32 + k] = in[32 + k];
    uint8_t* cw = w + 32 + l_qname;
    tr2chr(T, t, pos + 1, pos + l_seq, new_pos, cw, has_n);
    // bin from bam_endpos (sam.c:336-342): pos + reference length, which is pos itself for a CIGAR of insertions only
    int64_t rlen = 0;
    for (int k = 0; k < nc; ++k) {
        const uint32_t c = rd32(cw + 4 * k), op = c & 15;
        if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += c >> 4;
    }
    w[8] = (uint8_t)l_qname;
    w[9] = 255;
    wr16(w + 10, (uint16_t)reg2bin(new_pos, new_pos + rlen));
    wr16(w + 12, (uint16_t)nc);
    wr16(w + 14, flag);
    // sequence and qualities, complement-reversed on '-' (flipSeq / flipQual)
    uint8_t* os = cw + 4 * nc;
    uint8_t* oq = os + (l_seq + 1) / 2;
    if (minus) {
        for (int32_t i = 0; i < l_seq; i += 2) {
            uint8_t code = 0;
            for (int h = 0; h < 2 && i + h < l_seq; ++h) {
                const int j = l_seq - 1 - (i + h);
                const uint8_t b = (seq[j >> 1] >> ((j & 1) ? 0 : 4)) & 15;
                uint8_t c;
                switch (b) {
                    case 1: c = 8; break; case 2: c = 4; break; case 4: c = 2; break; case 8: c = 1; break; case 15: c = 15; break;
                    default: r.bad = kBadBase; return r;
                }
                code |= c << (h ? 0 : 4);
            }
            os[i >> 1] = code;
        }
        for (int32_t i = 0; i < l_seq; ++i) oq[i] = qual[l_seq - 1 - i];
    } else {
        for (int32_t i = 0; i < (l_seq + 1) / 2; ++i) os[i] = seq[i];
        for (int32_t i = 0; i < l_seq; ++i) oq[i] = qual[i];
    }
    // optional fields in order, without the first XS; MD rewritten on '-'
    uint8_t* oa = oq + l_seq;
    for (const uint8_t* a = aux; a < aux_end;) {
        const int len = aux_len(a + 2, aux_end);
        if (a != xs) {
            if (a == zw) r.zw = (int32_t)(oa - o);
            if (a == md && minus && a[2] == 'Z') {
                oa[0] = a[0]; oa[1] = a[1]; oa[2] = 'Z';
                const int l = len - 2;   // value bytes before the NUL
                md_flip(a + 3, oa + 3, l);
                oa[3 + l] = 0;
            } else {
                for (int k = 0; k < 2 + len; ++k) oa[k] = a[k];
            }
            oa += 2 + len;
        }
        a += 2 + len;
    }
    if (has_n) { oa[0] = 'X'; oa[1] = 'S'; oa[2] = 'A'; oa[3] = minus ? '-' : '+'; }
    return r;
}

__global__ void gbam_convert_kernel(Tables T, Batch B, uint8_t* __restrict__ conv, uint64_t* __restrict__ conv_off,
                                    int32_t* __restrict__ zw, float* __restrict__ prb, unsigned long long* err, bool write) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= B.n_units) return;
    const int t = B.unit_tr[u];
    if (!write) conv_off[u] = 0;
    if (t == 0) return;
    const uint32_t r0 = B.unit_rec[u], nr = B.unit_rec[u + 1] - r0;
    uint8_t* o = write ? conv + conv_off[u] : nullptr;
    uint64_t bytes = 0;
    int32_t pos[2] = {0, 0}, zwo[2] = {-1, -1};
    float p0 = 1.0f;
    for (uint32_t m = 0; m < nr; ++m) {
        const uint8_t* in = B.data + B.rec_off[r0 + m];
        const Conv c = convert(T, t, in + 4, rd32(in), o ? o + bytes : nullptr);
        if (c.bad) { flag_bad(err, u, c.bad); return; }
        if (m == 0) p0 = c.prb;
        pos[m] = c.pos;
        zwo[m] = c.zw < 0 ? -1 : (int32_t)(bytes + c.zw);
        bytes += c.bytes;
    }
    if (!write) { conv_off[u] = bytes; return; }
    if (nr == 2) {   // b->core.mpos = b2->core.pos and back (BamConverter.h:130-133)
        wr32(o + 4 + 24, (uint32_t)pos[1]);
        wr32(o + rd32(o) + 4 + 4 + 24, (uint32_t)pos[0]);
    }
    zw[2 * u] = zwo[0];
    zw[2 * u + 1] = zwo[1];
    prb[u] = p0;
}

// SingleEndT::compare (bc_aux.h:17-36) on two converted records (pointers at their block_size)
__device__ __forceinline__ int cmp_rec(const uint8_t* a, const uint8_t* b) {
    const int32_t ta = (int32_t)rd32(a + 4), tb = (int32_t)rd32(b + 4);
    if (ta != tb) return ta < tb ? -1 : 1;
    const int32_t pa = (int32_t)rd32(a + 8), pb = (int32_t)rd32(b + 8);
    if (pa != pb) return pa < pb ? -1 : 1;
    const int ra = (rd16(a + 18) >> 4) & 1, rb = (rd16(b + 18) >> 4) & 1;
    if (ra != rb) return ra < rb ? -1 : 1;
    const uint32_t na = rd16(a + 16), nb = rd16(b + 16);
    if (na != nb) return na < nb ? -1 : 1;
    const uint8_t* ca = a + 4 + 32 + a[12];
    const uint8_t* cb = b + 4 + 32 + b[12];
    for (uint32_t i = 0; i < na; ++i) {
        const uint32_t x = rd32(ca + 4 * i), y = rd32(cb + 4 * i);
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

struct UnitCmp {   // (group, mate 1's key, mate 2's key); PairedEndT::operator< (bc_aux.h:46-49)
    const uint32_t* group;
    const int32_t* tr;
    const uint32_t* unit_rec;
    const uint8_t* conv;
    const uint64_t* conv_off;
    __device__ int cmp(uint32_t a, uint32_t b) const {
        if (group[a] != group[b]) return group[a] < group[b] ? -1 : 1;
        if (tr[a] == 0 || tr[b] == 0) return 0;   // an unmapped unit is alone in its group
        const uint8_t* pa = conv + conv_off[a];
        const uint8_t* pb = conv + conv_off[b];
        const int c = cmp_rec(pa, pb);
        if (c || unit_rec[a + 1] - unit_rec[a] < 2) return c;
        return cmp_rec(pa + 4 + rd32(pa), pb + 4 + rd32(pb));
    }
    __device__ bool operator()(const uint32_t& a, const uint32_t& b) const { return cmp(a, b) < 0; }
};

__global__ void gbam_iota_kernel(uint32_t* keys, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keys[i] = i;
}

__global__ void gbam_heads_kernel(UnitCmp C, const uint32_t* __restrict__ keys, uint32_t n, uint8_t* __restrict__ head) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) head[i] = i == 0 || C.cmp(keys[i - 1], keys[i]) != 0;
}

// one thread per run head: the float sum of the run's ZW in input order (CollapseMap::insert), MAPQ, the output size
__global__ void gbam_collapse_kernel(Tables T, Batch B, const uint32_t* __restrict__ keys, const uint8_t* __restrict__ head,
                                     const float* __restrict__ prb, const uint64_t* __restrict__ conv_off,
                                     const uint8_t* __restrict__ conv, const int32_t* __restrict__ zw,
                                     float* __restrict__ run_prb, uint64_t* __restrict__ out_size, unsigned long long* err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.n_units) return;
    if (!head[i]) { out_size[i] = 0; return; }
    const uint32_t u = keys[i];
    const uint32_t r0 = B.unit_rec[u], nr = B.unit_rec[u + 1] - r0;
    if (B.unit_tr[u] == 0) {
        uint64_t bytes = 0;
        for (uint32_t m = 0; m < nr; ++m) bytes += 4 + rd32(B.data + B.rec_off[r0 + m]);
        out_size[i] = bytes;
        return;
    }
    float s = prb[u];
    for (uint32_t j = i + 1; j < B.n_units && !head[j]; ++j) s = __fadd_rn(s, prb[keys[j]]);
    run_prb[i] = s;
    if (zw[2 * u] >= 0 && !(s >= 0.0f)) flag_bad(err, u, kBadPrb);
    if (nr == 2 && zw[2 * u] >= 0 && zw[2 * u + 1] < 0) flag_bad(err, u, kBadMateZw);
    const uint8_t* c = conv + conv_off[u];
    out_size[i] = nr == 2 ? 8 + (uint64_t)rd32(c) + rd32(c + 4 + rd32(c)) : 4 + (uint64_t)rd32(c);
}

// writeCollapsedLines (BamConverter.h:193-219): the kept unit with ZW := the run's sum and MAPQ from it when mate 1 has
// ZW (MAPQ stays 255 otherwise); mate 2 takes mate 1's MAPQ and ZW
__global__ void gbam_emit_kernel(Tables T, Batch B, const uint32_t* __restrict__ keys, const uint8_t* __restrict__ head,
                                 const float* __restrict__ run_prb, const uint64_t* __restrict__ conv_off,
                                 const uint8_t* __restrict__ conv, const int32_t* __restrict__ zw,
                                 const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.n_units || !head[i]) return;
    const uint32_t u = keys[i];
    const uint32_t r0 = B.unit_rec[u], nr = B.unit_rec[u + 1] - r0;
    uint8_t* o = out + out_off[i];
    if (B.unit_tr[u] == 0) {
        for (uint32_t m = 0; m < nr; ++m) {
            const uint8_t* in = B.data + B.rec_off[r0 + m];
            const uint32_t n = 4 + rd32(in);
            for (uint32_t k = 0; k < n; ++k) o[k] = in[k];
            o += n;
        }
        return;
    }
    const uint8_t* c = conv + conv_off[u];
    const uint32_t n1 = 4 + rd32(c);
    const uint32_t n = nr == 2 ? n1 + 4 + rd32(c + n1) : n1;
    for (uint32_t k = 0; k < n; ++k) o[k] = c[k];
    if (zw[2 * u] < 0) return;
    const float s = run_prb[i];
    const uint32_t bits = __float_as_uint(s);
    int mapq = 0;
    for (int m = 1; m <= 100; ++m) mapq += s >= T.mapq_prb[m];
    wr32(o + zw[2 * u] + 3, bits);
    o[4 + 9] = (uint8_t)mapq;
    if (nr == 2) {
        if (zw[2 * u + 1] >= 0) wr32(o + zw[2 * u + 1] + 3, bits);
        o[n1 + 4 + 9] = (uint8_t)mapq;
    }
}

template <class T>
int grow(GbamState& S, T** p, size_t& have, size_t need) {
    if (need <= have && *p) return 0;
    if (*p) cudaFree(*p);
    *p = nullptr;
    have = std::max<size_t>(need + need / 4, 1024);
    RB_CUDA(cudaMalloc((void**)p, have * sizeof(T)));
    return 0;
}

template <class T>
int realloc_n(T** p, size_t n) {
    if (*p) cudaFree(*p);
    *p = nullptr;
    RB_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
    return 0;
}

int upload_tables(rsem_b200_ctx* ctx, GbamState& S, const rsem_b200_gbam_tables* t) {
    const int M = t->M;
    const int64_t E = t->exon_off[M + 1];
    auto up = [&](auto** dst, const auto* src, size_t n) -> int {
        using V = std::remove_pointer_t<std::remove_reference_t<decltype(*dst)>>;
        if (*dst) cudaFree(*dst);
        RB_CUDA(cudaMalloc((void**)dst, std::max<size_t>(n, 1) * sizeof(V)));
        if (n) RB_CUDA(cudaMemcpyAsync(*dst, src, n * sizeof(V), cudaMemcpyHostToDevice, ctx->stream));
        return 0;
    };
    int rc;
    if ((rc = up(&S.out_tid, t->out_tid, M + 1)) || (rc = up(&S.minus, t->minus, M + 1)) || (rc = up(&S.length, t->length, M + 1)) ||
        (rc = up(&S.exon_off, t->exon_off, M + 2)) || (rc = up(&S.exon_start, t->exon_start, E)) ||
        (rc = up(&S.exon_end, t->exon_end, E)) || (rc = up(&S.mapq_prb, t->mapq_prb, 101)))
        return rc;
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    S.tables_key = t;
    return 0;
}

const char* bad_text(unsigned why) {
    switch (why) {
        case kBadBase: return "a base code other than A, C, G, T or N (reference: assert(false) in flipSeq)";
        case kBadPos: return "a negative genomic position (reference: assert(core_pos >= 0))";
        case kBadExon: return "an alignment outside the transcript's exons (reference: assert(i < s) in tr2chr)";
        case kBadChr: return "a transcript whose sequence name is not in the chrlist file (reference: assert(iter != refmap.end()))";
        case kBadMateZw: return "mate 1 has a ZW tag and mate 2 has none";
        case kBadPrb: return "a ZW sum that is negative or not a number";
        default: return "an optional field of unknown type";
    }
}

}  // namespace

void gbam_free(rsem_b200_ctx* ctx) {
    GbamState* S = ctx->gbam;
    if (!S) return;
    void* ptrs[] = {S->out_tid, S->minus, S->length, S->exon_off, S->exon_start, S->exon_end, S->mapq_prb, S->data, S->conv,
                    S->out, S->head, S->rec_off, S->conv_off, S->out_off, S->unit_rec, S->unit_group, S->keys, S->unit_tr,
                    S->zw, S->prb, S->run_prb, S->temp, S->err};
    for (void* p : ptrs) if (p) cudaFree(p);
    for (auto& e : S->ev) if (e) cudaEventDestroy(e);
    delete S;
    ctx->gbam = nullptr;
}

int gbam_convert(rsem_b200_ctx* ctx, const rsem_b200_gbam_tables* t, const rsem_b200_gbam_batch* b, uint8_t* out,
                 uint64_t out_cap, uint64_t* out_bytes, rsem_b200_gbam_stats* stats) {
    if (!ctx->gbam) {
        ctx->gbam = new GbamState;
        RB_CUDA(cudaEventCreate(&ctx->gbam->ev[0]));
        RB_CUDA(cudaEventCreate(&ctx->gbam->ev[1]));
        RB_CUDA(cudaMalloc((void**)&ctx->gbam->err, sizeof(unsigned long long)));
    }
    GbamState& S = *ctx->gbam;
    int rc;
    if (S.tables_key != t && (rc = upload_tables(ctx, S, t))) return rc;
    rsem_b200_gbam_stats st{0.0, 0, -1};
    *out_bytes = 0;
    const uint32_t n = (uint32_t)b->n_units;
    if (n == 0) {
        if (stats) *stats = st;
        return 0;
    }
    const cudaStream_t s = ctx->stream;
    size_t rec_have = S.sz_rec, unit_have = S.sz_unit;
    if ((rc = grow(S, &S.data, S.sz_data, b->n_bytes))) return rc;
    if (b->n_records > rec_have || !S.rec_off) {
        size_t h = rec_have;
        if ((rc = grow(S, &S.rec_off, h, b->n_records))) return rc;
        S.sz_rec = h;
    }
    if (n + 1 > unit_have) {   // every per-unit array holds S.sz_unit entries, zw twice that
        const size_t cap = std::max<size_t>((n + 1) + (n + 1) / 4, 1024);
        if ((rc = realloc_n(&S.unit_rec, cap)) || (rc = realloc_n(&S.unit_group, cap)) || (rc = realloc_n(&S.unit_tr, cap)) ||
            (rc = realloc_n(&S.keys, cap)) || (rc = realloc_n(&S.conv_off, cap)) || (rc = realloc_n(&S.out_off, cap)) ||
            (rc = realloc_n(&S.head, cap)) || (rc = realloc_n(&S.prb, cap)) || (rc = realloc_n(&S.run_prb, cap)) ||
            (rc = realloc_n(&S.zw, 2 * cap)))
            return rc;
        S.sz_unit = cap;
    }
    RB_CUDA(cudaEventRecord(S.ev[0], s));
    RB_CUDA(cudaMemcpyAsync(S.data, b->data, b->n_bytes, cudaMemcpyHostToDevice, s));
    RB_CUDA(cudaMemcpyAsync(S.rec_off, b->rec_off, b->n_records * 8, cudaMemcpyHostToDevice, s));
    RB_CUDA(cudaMemcpyAsync(S.unit_rec, b->unit_rec, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, s));
    RB_CUDA(cudaMemcpyAsync(S.unit_group, b->unit_group, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    RB_CUDA(cudaMemcpyAsync(S.unit_tr, b->unit_tr, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    RB_CUDA(cudaMemsetAsync(S.err, 0xff, sizeof(unsigned long long), s));
    Tables T{S.out_tid, S.minus, S.length, S.exon_off, S.exon_start, S.exon_end, S.mapq_prb};
    Batch B{S.data, S.rec_off, S.unit_rec, S.unit_group, S.unit_tr, n};
    const unsigned grid = (n + kThreads - 1) / kThreads;

    // sizes, scan, convert
    gbam_convert_kernel<<<grid, kThreads, 0, s>>>(T, B, nullptr, S.conv_off, S.zw, S.prb, S.err, false);
    RB_CUDA(cudaGetLastError());
    size_t tb1 = 0, tb2 = 0, tb3 = 0;
    UnitCmp C{S.unit_group, S.unit_tr, S.unit_rec, nullptr, S.conv_off};
    RB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb1, S.conv_off, S.conv_off, n + 1, s));
    RB_CUDA(cub::DeviceMergeSort::StableSortKeys(nullptr, tb2, S.keys, n, C, s));
    RB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb3, S.out_off, S.out_off, n + 1, s));
    if ((rc = grow(S, (uint8_t**)&S.temp, S.sz_temp, std::max({tb1, tb2, tb3})))) return rc;
    // conv_off[n] is the total after the scan: the sizes pass leaves it 0
    RB_CUDA(cudaMemsetAsync(S.conv_off + n, 0, 8, s));
    RB_CUDA(cub::DeviceScan::ExclusiveSum(S.temp, tb1, S.conv_off, S.conv_off, n + 1, s));
    uint64_t conv_total = 0;
    unsigned long long err = 0;
    // a unit flagged by a pass is not read by the passes after it: the call stops at the next check
    auto check = [&]() -> int {
        RB_CUDA(cudaMemcpyAsync(&err, S.err, sizeof err, cudaMemcpyDeviceToHost, s));
        RB_CUDA(cudaStreamSynchronize(s));
        if (err == ~0ull) return 0;
        st.bad_unit = (int64_t)(err >> 8);
        if (stats) *stats = st;
        set_error(std::string("gbam_convert: ") + bad_text((unsigned)(err & 255)));
        return RSEM_B200_ERR_ARG;
    };
    RB_CUDA(cudaMemcpyAsync(&conv_total, S.conv_off + n, 8, cudaMemcpyDeviceToHost, s));
    if ((rc = check())) return rc;
    if ((rc = grow(S, &S.conv, S.sz_conv, conv_total))) return rc;
    gbam_convert_kernel<<<grid, kThreads, 0, s>>>(T, B, S.conv, S.conv_off, S.zw, S.prb, S.err, true);
    RB_CUDA(cudaGetLastError());
    if ((rc = check())) return rc;

    // stable sort by (group, key), run heads, sums, sizes
    C.conv = S.conv;
    gbam_iota_kernel<<<grid, kThreads, 0, s>>>(S.keys, n);
    RB_CUDA(cudaGetLastError());
    RB_CUDA(cub::DeviceMergeSort::StableSortKeys(S.temp, tb2, S.keys, n, C, s));
    gbam_heads_kernel<<<grid, kThreads, 0, s>>>(C, S.keys, n, S.head);
    RB_CUDA(cudaGetLastError());
    gbam_collapse_kernel<<<grid, kThreads, 0, s>>>(T, B, S.keys, S.head, S.prb, S.conv_off, S.conv, S.zw, S.run_prb, S.out_off, S.err);
    RB_CUDA(cudaGetLastError());
    RB_CUDA(cudaMemsetAsync(S.out_off + n, 0, 8, s));
    RB_CUDA(cub::DeviceScan::ExclusiveSum(S.temp, tb3, S.out_off, S.out_off, n + 1, s));
    uint64_t out_total = 0;
    RB_CUDA(cudaMemcpyAsync(&out_total, S.out_off + n, 8, cudaMemcpyDeviceToHost, s));
    ctx->launches += 6;
    if ((rc = check())) return rc;
    if (out_total > out_cap) {
        set_error("gbam_convert: the output buffer is too small");
        return RSEM_B200_ERR_ARG;
    }
    if ((rc = grow(S, &S.out, S.sz_out, out_total))) return rc;
    gbam_emit_kernel<<<grid, kThreads, 0, s>>>(T, B, S.keys, S.head, S.run_prb, S.conv_off, S.conv, S.zw, S.out_off, S.out);
    RB_CUDA(cudaGetLastError());
    ctx->launches += 1;
    RB_CUDA(cudaMemcpyAsync(out, S.out, out_total, cudaMemcpyDeviceToHost, s));
    RB_CUDA(cudaEventRecord(S.ev[1], s));
    RB_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, S.ev[0], S.ev[1]);
    st.device_ms = ms;
    *out_bytes = out_total;
    if (stats) *stats = st;
    return 0;
}

}  // namespace rsem_b200
