// mksnap_inflate_core.h -- the gzip / DEFLATE logic of the engine's gunzip (mksnap_gunzip_*), written once as
// __host__ __device__ code: the kernels of mksnap_inflate.cuh run it on the H100, the engine's host side runs the link
// step, and the CPU mock of the engine (tests/mock_engine/mock_mksnap.cpp) compiles the same file with g++, so the CPU
// tests fuzz the code that runs on the GPU.
//
// Segments.  A blob is cut at candidate starts (CAND_FLUSH, CAND_MEMBER below): the byte after every `00 00 FF FF` (the empty stored block
// a sync or full flush ends with) and the body start of every byte-aligned member header the parser accepts, so that
// the members of a bgzip / eStargz / concatenated blob decode in parallel.  decode_segment() decodes from one start
// until a block ends exactly on a later candidate, or the final block of the member ends.  A candidate that is not a
// true start (a pattern inside compressed data) is harmless: decoding from it fails or is never linked, and a block
// that happens to end on it is a true block boundary, where cutting a segment is exact.  Decoding from a start that is really a
// block boundary is exact without the output before it, except for back-references into the 32 KiB before the
// segment: in write mode those bytes become markers (0x8000 | index into that 32 KiB), which resolve_segment_tail()
// and resolve_symbol() replace once the previous segments are known.
//
// Indexed open (mksnap_gunzip_open_indexed): the same decoder, link and candidate rule at bit granularity
// (decode_segment_t<true>, link_feed<true>), so that a caller's points -- DEFLATE block headers at any bit -- are
// candidates like the scanned ones.  Count decodes record a block start about every SPLIT_OUT output bytes (Recorder),
// and split_segments() cuts each long linked segment at the records of its own decode: those are true block starts of
// the chain with known output offsets, so a single member without flush points decodes in parallel after one serial
// count pass, and the cuts are the index a later open of the same blob takes as points.
//
// Acceptance is zlib's raw inflate (stored / fixed / dynamic blocks, inftrees' rules on over-subscribed and incomplete
// code sets, 286/287 and 30/31 invalid, a distance before the member start invalid) and Go's compress/gzip header and
// multistream rules (FNAME / FCOMMENT at most 511 bytes, FHCRC checked, anything after a member that is not a member
// header is an error, reserved flag bits ignored).
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#if defined(__CUDACC__)
#define MKI_HD __host__ __device__
#else
#define MKI_HD
#endif

namespace mki {

constexpr uint32_t WSIZE = 32768;    // DEFLATE window
constexpr uint16_t MARK = 0x8000u;   // write-mode symbol: MARK | index into the 32 KiB before the segment
constexpr uint32_t FAST = 9;         // bits of the direct Huffman lookup
constexpr uint32_t NO_LIMIT = 0xFFFFFFFFu;
constexpr uint32_t K_PASS = 4;       // candidates a speculative decode may pass before it stops (DESIGN.md section 5)

enum : int32_t {
    SEG_ERR = -1,     // malformed data
    SEG_CAND = 1,     // a non-final block ended on a candidate start: the segment ends there
    SEG_FINAL = 2,    // the final block ended: end = first byte after it (the member trailer)
    SEG_SUSPEND = 3,  // a speculative decode passed more than K candidates and stopped; redo it if it is on the chain
};

struct SegRes {
    uint64_t end;      // byte offset where the segment ends (SEG_CAND / SEG_FINAL)
    uint64_t out_len;  // bytes it decodes to
    uint64_t consumed; // input bytes the decode went through (work measure; any status)
    int32_t status;
    uint32_t reserved;
};

struct Huff {
    uint16_t count[16];
    uint16_t sym[288];
    uint16_t fast[1u << FAST]; // (len << 9) | sym, 0 = take the bit-serial path
};

struct Tables {
    Huff lit, dist;
    uint16_t lens[320];
};

// ---- bit reader ---------------------------------------------------------------------------------------------------
struct Bits {
    const uint8_t *in;
    uint64_t n;   // input length
    uint64_t pos; // next byte to load
    uint64_t bb;  // bit buffer, LSB first
    uint32_t bc;  // bits in bb
    MKI_HD void refill()
    {
        while (bc <= 56 && pos < n) {
            bb |= (uint64_t)in[pos++] << bc;
            bc += 8;
        }
    }
    MKI_HD uint64_t bitpos() const { return pos * 8 - bc; }
    // false when the input ends first
    MKI_HD bool get(uint32_t k, uint32_t *v)
    {
        if (bc < k) {
            refill();
            if (bc < k)
                return false;
        }
        *v = (uint32_t)(bb & ((1ull << k) - 1));
        bb >>= k;
        bc -= k;
        return true;
    }
    MKI_HD void align_byte() // stored block: drop to the byte boundary, then reload from there
    {
        const uint64_t p = (bitpos() + 7) / 8;
        pos = p;
        bb = 0;
        bc = 0;
    }
};

// Canonical code from lengths.  Returns 0, or -1 where zlib's inflate_table refuses the set: over-subscribed, or
// incomplete unless `allow_incomplete` and the longest code has length 1 (a set with no codes at all is accepted; a
// symbol decoded from it is an error).
MKI_HD inline int build_huff(Huff *h, const uint16_t *len, uint32_t n, bool allow_incomplete)
{
    for (int l = 0; l < 16; ++l)
        h->count[l] = 0;
    for (uint32_t s = 0; s < n; ++s)
        h->count[len[s]]++;
    uint32_t maxl = 0;
    for (uint32_t l = 1; l < 16; ++l)
        if (h->count[l])
            maxl = l;
    for (uint32_t i = 0; i < (1u << FAST); ++i)
        h->fast[i] = 0;
    if (maxl == 0)
        return 0;
    int32_t left = 1;
    for (uint32_t l = 1; l < 16; ++l) {
        left <<= 1;
        left -= h->count[l];
        if (left < 0)
            return -1;
    }
    if (left > 0 && (!allow_incomplete || maxl != 1))
        return -1;
    uint16_t offs[16];
    offs[1] = 0;
    for (uint32_t l = 1; l < 15; ++l)
        offs[l + 1] = (uint16_t)(offs[l] + h->count[l]);
    for (uint32_t s = 0; s < n; ++s)
        if (len[s])
            h->sym[offs[len[s]]++] = (uint16_t)s;
    // direct table: every code of length <= FAST, bit-reversed (DEFLATE sends Huffman codes MSB first)
    uint32_t code = 0, idx = 0;
    for (uint32_t l = 1; l <= FAST; ++l) {
        for (uint32_t k = 0; k < h->count[l]; ++k, ++code, ++idx) {
            uint32_t r = 0;
            for (uint32_t b = 0; b < l; ++b)
                r |= ((code >> b) & 1u) << (l - 1 - b);
            for (uint32_t f = r; f < (1u << FAST); f += 1u << l)
                h->fast[f] = (uint16_t)((l << 9) | h->sym[idx]);
        }
        code <<= 1;
    }
    return 0;
}

// next symbol, or -1 (input ended, or a code the set does not have)
MKI_HD inline int32_t decode_sym(Bits &b, const Huff &h)
{
    if (b.bc < 15)
        b.refill();
    const uint32_t e = h.fast[b.bb & ((1u << FAST) - 1)];
    if (e) {
        const uint32_t l = e >> 9;
        if (l > b.bc)
            return -1;
        b.bb >>= l;
        b.bc -= l;
        return (int32_t)(e & 511u);
    }
    int32_t code = 0, first = 0, index = 0;
    for (uint32_t l = 1; l < 16; ++l) {
        if (b.bc == 0)
            return -1;
        code |= (int32_t)(b.bb & 1u);
        b.bb >>= 1;
        b.bc -= 1;
        const int32_t c = h.count[l];
        if (code - c < first)
            return h.sym[index + (code - first)];
        index += c;
        first += c;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

MKI_HD inline void fixed_tables(Tables *t)
{
    uint32_t s = 0;
    for (; s < 144; ++s) t->lens[s] = 8;
    for (; s < 256; ++s) t->lens[s] = 9;
    for (; s < 280; ++s) t->lens[s] = 7;
    for (; s < 288; ++s) t->lens[s] = 8;
    build_huff(&t->lit, t->lens, 288, false);
    for (s = 0; s < 32; ++s) t->lens[s] = 5;
    build_huff(&t->dist, t->lens, 32, false); // codes 30 and 31 decode, and the caller refuses them
}

MKI_HD inline int dynamic_tables(Bits &b, Tables *t)
{
    static const uint8_t ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    uint32_t hlit, hdist, hclen, v;
    if (!b.get(5, &hlit) || !b.get(5, &hdist) || !b.get(4, &hclen))
        return -1;
    const uint32_t nlen = hlit + 257, ndist = hdist + 1, ncode = hclen + 4;
    if (nlen > 286 || ndist > 30)
        return -1;
    for (uint32_t i = 0; i < 19; ++i)
        t->lens[i] = 0;
    for (uint32_t i = 0; i < ncode; ++i) {
        if (!b.get(3, &v))
            return -1;
        t->lens[ORDER[i]] = (uint16_t)v;
    }
    Huff &cl = t->lit; // the code-length code lives in the lit/len table until the lengths are read
    if (build_huff(&cl, t->lens, 19, false) != 0)
        return -1;
    uint16_t ll[320];
    uint32_t i = 0;
    while (i < nlen + ndist) {
        const int32_t s = decode_sym(b, cl);
        if (s < 0)
            return -1;
        if (s < 16) {
            ll[i++] = (uint16_t)s;
            continue;
        }
        uint32_t rep, val = 0;
        if (s == 16) {
            if (i == 0 || !b.get(2, &rep))
                return -1;
            val = ll[i - 1];
            rep += 3;
        } else if (s == 17) {
            if (!b.get(3, &rep))
                return -1;
            rep += 3;
        } else {
            if (!b.get(7, &rep))
                return -1;
            rep += 11;
        }
        if (i + rep > nlen + ndist)
            return -1;
        while (rep--)
            ll[i++] = (uint16_t)val;
    }
    if (ll[256] == 0) // no end-of-block code
        return -1;
    if (build_huff(&t->lit, ll, nlen, true) != 0)
        return -1;
    if (build_huff(&t->dist, ll + nlen, ndist, true) != 0)
        return -1;
    return 0;
}

// first candidate index with cand[i] > x
MKI_HD inline uint64_t upper_bound(const uint64_t *cand, uint64_t n, uint64_t x)
{
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if (cand[mid] <= x)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// ---- block-start records (mksnap_gunzip_open_indexed) ----------------------------------------------------------------
// A count decode records the first block header at least SPLIT_OUT output bytes after its start or after its previous
// record: its bit offset and its output offset in the segment.  Such a record is a true block start of that decode, so
// a linked segment can be cut there without a second pass.  Records of all decodes share one bounded buffer; those past
// its capacity are dropped, which only leaves a segment longer.
constexpr uint64_t SPLIT_OUT = 1ull << 20;
constexpr uint64_t REC_CAP = 1ull << 16; // records one open keeps (24 B each: 1.5 MiB)

struct Rec {
    uint64_t from; // start bit of the decode that recorded it
    uint64_t bit;  // block header
    uint64_t out;  // output bytes of that decode before the block
};

struct Recorder {
    Rec *buf;
    unsigned long long *n; // records offered (may exceed cap)
    uint64_t cap;
    MKI_HD void put(uint64_t from, uint64_t bit, uint64_t out) const
    {
#if defined(__CUDA_ARCH__)
        const uint64_t k = atomicAdd(n, 1ull);
#else
        const uint64_t k = (*n)++;
#endif
        if (k < cap)
            buf[k] = Rec{from, bit, out};
    }
};

// Decode one segment from byte `start` of gz.
//   count mode (out == nullptr): nothing is written; the decode stops (SEG_SUSPEND) once it has passed more than K
//     candidates, so the speculative decodes of all candidates together read O(K * gz_len) bytes for any input.
//   write mode: out[j] = byte j of the segment, or MARK | (32768 + j - dist) for a byte that copies from before the
//     segment.  member_pos = output bytes of the member before the segment: a distance beyond that is an error.
//     out_cap bounds what is written.
//   BITS (mksnap_gunzip_open_indexed): `start`, the candidates and SegRes::end are bit offsets (SEG_FINAL: 8 times the
//     trailer's byte offset), and a count-mode decode given `rec` records block starts (Recorder).
template <bool BITS>
MKI_HD inline SegRes decode_segment_t(const uint8_t *gz, uint64_t gz_len, uint64_t start, const uint64_t *cand,
                                      uint64_t n_cand, uint32_t K, uint16_t *out, uint64_t out_cap, uint64_t member_pos,
                                      Tables *t, const Recorder *rec)
{
    static const uint16_t LBASE[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                       31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
    static const uint8_t LEXT[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    static const uint16_t DBASE[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                       193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
    static const uint8_t DEXT[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
    SegRes r = {0, 0, 0, SEG_ERR, 0};
    const uint64_t start_byte = BITS ? start / 8 : start;
    Bits b = {gz, gz_len, start_byte, 0, 0};
    uint64_t ci = upper_bound(cand, n_cand, start); // next candidate not yet passed
    uint64_t next_bits = ci < n_cand ? (BITS ? cand[ci] : cand[ci] * 8) : ~0ull;
    uint32_t passed = 0;
    uint64_t j = 0; // output position in the segment
    uint64_t rec_at = SPLIT_OUT; // output position from which the next block start is recorded
#define MKI_FAIL()                                  \
    do {                                            \
        r.consumed = (b.bitpos() + 7) / 8 - start_byte; \
        r.out_len = j;                              \
        return r;                                   \
    } while (0)
    // candidates strictly before bit position p are passed; true when the K limit stops the decode
#define MKI_PASS(p)                                                 \
    while ((p) > next_bits) {                                       \
        if (++passed > K) {                                         \
            r.status = SEG_SUSPEND;                                 \
            r.consumed = (BITS ? cand[ci] / 8 : cand[ci]) + 1 - start_byte; \
            r.out_len = j;                                          \
            return r;                                               \
        }                                                           \
        ++ci;                                                       \
        next_bits = ci < n_cand ? (BITS ? cand[ci] : cand[ci] * 8) : ~0ull; \
    }
    if (BITS && (start & 7)) {
        uint32_t v;
        if (!b.get((uint32_t)(start & 7), &v))
            MKI_FAIL();
    }
    for (;;) {
        if (BITS && rec && j >= rec_at) {
            rec->put(start, b.bitpos(), j);
            rec_at = j + SPLIT_OUT;
        }
        uint32_t final, type;
        if (!b.get(1, &final) || !b.get(2, &type))
            MKI_FAIL();
        if (type == 0) {
            b.align_byte();
            uint32_t ln, nl;
            if (!b.get(16, &ln) || !b.get(16, &nl) || ln != (~nl & 0xFFFFu))
                MKI_FAIL();
            const uint64_t p = b.bitpos() / 8; // the bit buffer holds whole bytes here
            if (p + ln > gz_len)
                MKI_FAIL();
            MKI_PASS(8 * (p + ln));
            if (out) {
                if (j + ln > out_cap)
                    MKI_FAIL();
                for (uint32_t k = 0; k < ln; ++k)
                    out[j + k] = gz[p + k];
            }
            j += ln;
            b.pos = p + ln;
            b.bb = 0;
            b.bc = 0;
        } else if (type == 3) {
            MKI_FAIL();
        } else {
            if (type == 1)
                fixed_tables(t);
            else if (dynamic_tables(b, t) != 0)
                MKI_FAIL();
            for (;;) {
                const int32_t s = decode_sym(b, t->lit);
                if (s < 0 || s > 285)
                    MKI_FAIL();
                if (s < 256) {
                    if (out) {
                        if (j >= out_cap)
                            MKI_FAIL();
                        out[j] = (uint16_t)s;
                    }
                    ++j;
                } else if (s == 256) {
                    break;
                } else {
                    uint32_t e, len, dist;
                    if (!b.get(LEXT[s - 257], &e))
                        MKI_FAIL();
                    len = LBASE[s - 257] + e;
                    const int32_t ds = decode_sym(b, t->dist);
                    if (ds < 0 || ds > 29 || !b.get(DEXT[ds], &e))
                        MKI_FAIL();
                    dist = DBASE[ds] + e;
                    if (out) {
                        if (dist > member_pos + j || j + len > out_cap)
                            MKI_FAIL();
                        for (uint32_t k = 0; k < len; ++k, ++j) {
                            const int64_t src = (int64_t)j - (int64_t)dist;
                            out[j] = src >= 0 ? out[src] : (uint16_t)(MARK | (uint32_t)(WSIZE + src));
                        }
                    } else {
                        j += len;
                    }
                }
                MKI_PASS(b.bitpos());
            }
        }
        const uint64_t bp = b.bitpos();
        if (final) {
            r.status = SEG_FINAL;
            r.end = BITS ? (bp + 7) / 8 * 8 : (bp + 7) / 8;
            break;
        }
        MKI_PASS(bp);
        if (bp == next_bits) {
            r.status = SEG_CAND;
            r.end = BITS ? bp : bp / 8;
            break;
        }
    }
#undef MKI_PASS
#undef MKI_FAIL
    r.out_len = j;
    r.consumed = BITS ? (r.end - start) / 8 : r.end - start;
    return r;
}

MKI_HD inline SegRes decode_segment(const uint8_t *gz, uint64_t gz_len, uint64_t start, const uint64_t *cand,
                                    uint64_t n_cand, uint32_t K, uint16_t *out, uint64_t out_cap, uint64_t member_pos,
                                    Tables *t)
{
    return decode_segment_t<false>(gz, gz_len, start, cand, n_cand, K, out, out_cap, member_pos, t, nullptr);
}

// ---- gzip framing (RFC 1952, with Go compress/gzip's limits) -------------------------------------------------------
MKI_HD inline uint32_t crc32_update(uint32_t c, const uint8_t *p, uint64_t n) // small header runs only
{
    c = ~c;
    for (uint64_t i = 0; i < n; ++i) {
        c ^= p[i];
        for (int k = 0; k < 8; ++k)
            c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
    }
    return ~c;
}

// Member header at `off`: returns the offset of the member body, or -1 (not a valid header, or it is cut short).
// check_hcrc = false skips the FHCRC comparison (the two bytes are still required): the candidate scan, where a header
// with FEXTRA would otherwise cost a bitwise CRC over up to 64 KiB at each of up to gz_len / 3 offsets.
MKI_HD inline int64_t parse_header(const uint8_t *gz, uint64_t gz_len, uint64_t off, bool check_hcrc = true)
{
    if (off + 10 > gz_len || gz[off] != 0x1f || gz[off + 1] != 0x8b || gz[off + 2] != 8)
        return -1;
    const uint8_t flg = gz[off + 3];
    uint64_t p = off + 10;
    if (flg & 4) { // FEXTRA
        if (p + 2 > gz_len)
            return -1;
        const uint64_t xlen = gz[p] | ((uint64_t)gz[p + 1] << 8);
        p += 2;
        if (p + xlen > gz_len)
            return -1;
        p += xlen;
    }
    for (int f = 8; f <= 16; f <<= 1) { // FNAME, FCOMMENT: zero-terminated, at most 512 bytes with the terminator
        if (!(flg & f))
            continue;
        uint64_t i = 0;
        for (;; ++i) {
            if (i >= 512 || p + i >= gz_len)
                return -1;
            if (gz[p + i] == 0)
                break;
        }
        p += i + 1;
    }
    if (flg & 2) { // FHCRC: low 16 bits of the CRC-32 of the header bytes before it
        if (p + 2 > gz_len)
            return -1;
        const uint32_t want = gz[p] | ((uint32_t)gz[p + 1] << 8);
        if (check_hcrc && (crc32_update(0, gz + off, p - off) & 0xFFFFu) != want)
            return -1;
        p += 2;
    }
    return (int64_t)p;
}

// ---- candidate starts -----------------------------------------------------------------------------------------------
// Candidates are the offsets p, first_body < p <= gz_len, of either kind (both bits when both hold); first_body, the
// first member's body start, is candidate 0.  At most gz_len / 4 + gz_len / 3 + 1 of them: `00 00 FF FF` cannot
// overlap itself and `1f 8b 08` cannot overlap itself or it, and each header start gives one body start.
enum : uint8_t {
    CAND_FLUSH = 1,  // gz[p-4..p) == 00 00 FF FF
    CAND_MEMBER = 2, // p is the body start of a header at some q < p (member_body(q) == p)
};

MKI_HD inline bool flush_end(const uint8_t *gz, uint64_t p)
{
    return p >= 4 && gz[p - 1] == 0xFF && gz[p - 2] == 0xFF && gz[p - 3] == 0 && gz[p - 4] == 0;
}

// body start of a member header at q as the scan sees it (FHCRC not compared, see parse_header), or -1.  Bodies of
// headers at different q need not be in the order of q (FEXTRA can hold a header), nor distinct.
MKI_HD inline int64_t member_body(const uint8_t *gz, uint64_t gz_len, uint64_t q)
{
    if (q + 3 > gz_len || gz[q] != 0x1f || gz[q + 1] != 0x8b || gz[q + 2] != 8)
        return -1;
    return parse_header(gz, gz_len, q, false);
}

// ---- link: the true chain of segments through the speculative results --------------------------------------------
struct Seg {
    uint64_t start, end; // compressed byte range (bit range after an indexed open)
    uint64_t out_off;    // offset in the decompressed stream
    uint64_t out_len;
    uint64_t member_pos; // output bytes of its member before it
    uint32_t member;
    uint32_t final;      // last segment of its member
};

struct Member {
    uint64_t out_off, out_len; // decompressed range
    uint32_t crc, isize;       // trailer
};

struct LinkState {
    uint64_t pos;       // start of the next segment (a bit offset in BITS mode)
    uint64_t out;       // output bytes so far
    uint64_t mpos;      // output bytes of the current member so far
    uint32_t member;    // index of the current member
    uint32_t done;
};

enum : int { LINK_NEXT = 0, LINK_DONE = 1, LINK_ERR = -1 };

// Start at the first member's header.  LINK_ERR: no valid member header at offset 0.  BITS: positions are bit offsets
// (decode_segment_t<true>).
template <bool BITS = false>
MKI_HD inline int link_start(LinkState *st, const uint8_t *gz, uint64_t gz_len)
{
    const int64_t body = parse_header(gz, gz_len, 0);
    *st = LinkState{0, 0, 0, 0, 0};
    if (body < 0)
        return LINK_ERR;
    st->pos = BITS ? (uint64_t)body * 8 : (uint64_t)body;
    return LINK_NEXT;
}

// Feed the result of the segment that starts at st->pos (a finished decode: SEG_CAND, SEG_FINAL or SEG_ERR).  Writes
// *seg, and *mem when the segment ends its member; returns LINK_NEXT (st->pos is the next start), LINK_DONE or
// LINK_ERR.  After a final segment the trailer is read and whatever follows must be the end of the blob or another
// member header.
template <bool BITS = false>
MKI_HD inline int link_feed(LinkState *st, const SegRes &r, const uint8_t *gz, uint64_t gz_len, Seg *seg, Member *mem,
                            bool *ended_member)
{
    *ended_member = false;
    if (r.status != SEG_CAND && r.status != SEG_FINAL)
        return LINK_ERR;
    *seg = Seg{st->pos, r.end, st->out, r.out_len, st->mpos, st->member, r.status == SEG_FINAL ? 1u : 0u};
    st->out += r.out_len;
    st->mpos += r.out_len;
    if (r.status == SEG_CAND) {
        st->pos = r.end;
        return LINK_NEXT;
    }
    const uint64_t t = BITS ? r.end / 8 : r.end;
    if (t + 8 > gz_len)
        return LINK_ERR;
    mem->out_off = st->out - st->mpos;
    mem->out_len = st->mpos;
    mem->crc = gz[t] | ((uint32_t)gz[t + 1] << 8) | ((uint32_t)gz[t + 2] << 16) | ((uint32_t)gz[t + 3] << 24);
    mem->isize = gz[t + 4] | ((uint32_t)gz[t + 5] << 8) | ((uint32_t)gz[t + 6] << 16) | ((uint32_t)gz[t + 7] << 24);
    *ended_member = true;
    if (t + 8 == gz_len) {
        st->done = 1;
        return LINK_DONE;
    }
    const int64_t body = parse_header(gz, gz_len, t + 8);
    if (body < 0)
        return LINK_ERR;
    st->pos = BITS ? (uint64_t)body * 8 : (uint64_t)body;
    st->mpos = 0;
    st->member++;
    return LINK_NEXT;
}

// The link over the count results (host only): from st->pos, take the result of the candidate that starts there, or
// else call redecode(pos, &r) for a decode without the K limit (a start that is no candidate, or whose count decode
// was suspended), and feed it to link_feed until the last member ends.  Returns LINK_DONE, LINK_ERR (st->member and
// st->pos name the place), or the nonzero rc of redecode, which must differ from both.
template <bool BITS, class Redecode>
inline int link_all(LinkState *st, const uint64_t *cand, const SegRes *res, uint64_t n, const uint8_t *gz,
                    uint64_t gz_len, Redecode &&redecode, std::vector<Seg> *segs, std::vector<Member> *mems)
{
    for (;;) {
        const uint64_t i = upper_bound(cand, n, st->pos);
        SegRes r;
        if (i > 0 && cand[i - 1] == st->pos && res[i - 1].status != SEG_SUSPEND) {
            r = res[i - 1];
        } else if (const int rc = redecode(st->pos, &r)) {
            return rc;
        }
        Seg seg;
        Member mem;
        bool ended = false;
        const int lk = link_feed<BITS>(st, r, gz, gz_len, &seg, &mem, &ended);
        if (lk == LINK_ERR)
            return LINK_ERR;
        segs->push_back(seg);
        if (ended)
            mems->push_back(mem);
        if (lk == LINK_DONE)
            return LINK_DONE;
    }
}

// ---- indexed open: the host steps around the count pass and the link --------------------------------------------------
// Candidates of an indexed open: the scanned byte candidates as bit offsets, merged with the caller's points (bit
// offsets, strictly ascending), without duplicates.
inline std::vector<uint64_t> merge_points(const std::vector<uint64_t> &byte_cand, const uint64_t *points, uint64_t n)
{
    std::vector<uint64_t> out;
    out.reserve(byte_cand.size() + n);
    uint64_t i = 0, k = 0;
    while (i < byte_cand.size() || k < n) {
        const uint64_t v = k == n || (i < byte_cand.size() && byte_cand[i] * 8 <= points[k]) ? byte_cand[i++] * 8 : points[k++];
        if (out.empty() || out.back() != v)
            out.push_back(v);
    }
    return out;
}

struct IndexCounts {
    uint64_t linked;   // given points that start a linked segment
    uint64_t recorded; // cuts taken from records
};

// After the link: every segment that decodes to more than SPLIT_OUT bytes is cut at the records of the decode the link
// followed (records with from == its start; a suspended count decode redone on the chain records the same blocks
// twice).  `cand` (bit candidates) gains the cuts, so that the write decode of each piece ends exactly at the next one;
// `index` gets the starts of the final segments that are not scanned candidates: the points worth giving a later open.
inline IndexCounts split_segments(std::vector<Seg> *segs, std::vector<Rec> recs, std::vector<uint64_t> *cand,
                                  const std::vector<uint64_t> &byte_cand, const uint64_t *points, uint64_t n_points,
                                  std::vector<uint64_t> *index)
{
    IndexCounts c{0, 0};
    std::sort(recs.begin(), recs.end(),
              [](const Rec &a, const Rec &b) { return a.from != b.from ? a.from < b.from : a.bit < b.bit; });
    std::vector<Seg> out;
    std::vector<uint64_t> cuts;
    for (const Seg &s : *segs) {
        if (std::binary_search(points, points + n_points, s.start))
            ++c.linked;
        uint64_t bit = s.start, o = 0;
        if (s.out_len > SPLIT_OUT) {
            auto it = std::lower_bound(recs.begin(), recs.end(), s.start,
                                       [](const Rec &r, uint64_t v) { return r.from < v; });
            for (; it != recs.end() && it->from == s.start; ++it) {
                if (it->bit <= bit || it->bit >= s.end || it->out <= o || it->out >= s.out_len)
                    continue;
                out.push_back(Seg{bit, it->bit, s.out_off + o, it->out - o, s.member_pos + o, s.member, 0});
                cuts.push_back(it->bit);
                bit = it->bit;
                o = it->out;
            }
        }
        out.push_back(Seg{bit, s.end, s.out_off + o, s.out_len - o, s.member_pos + o, s.member, s.final});
    }
    c.recorded = cuts.size();
    std::vector<uint64_t> merged(cand->size() + cuts.size());
    std::merge(cand->begin(), cand->end(), cuts.begin(), cuts.end(), merged.begin());
    cand->swap(merged);
    index->clear();
    for (const Seg &s : out)
        if (s.start % 8 || !std::binary_search(byte_cand.begin(), byte_cand.end(), s.start / 8))
            index->push_back(s.start);
    segs->swap(out);
    return c;
}

// ---- resolve ------------------------------------------------------------------------------------------------------
// A window holds whole segments back to back in `sym` (window-relative offsets); `hist` is the 32 KiB of output before
// the window (zero where the stream has none: no valid reference reaches there).  The byte a symbol at window offset
// `p` of the segment starting at window offset `o` stands for:
MKI_HD inline uint8_t resolve_symbol(const uint16_t *sym, const uint8_t *hist, uint64_t o, uint16_t v)
{
    if (!(v & MARK))
        return (uint8_t)v;
    const int64_t q = (int64_t)o - (int64_t)WSIZE + (int64_t)(v & 0x7FFFu); // window offset of the referenced byte
    return q >= 0 ? (uint8_t)sym[q] : hist[WSIZE + q];
}

// In segment order, the last 32 KiB of each segment are resolved in place (symbols become literals): every marker of a
// later segment then points at resolved symbols or into hist.  Within a segment the positions are independent, so a
// device runs them in parallel (stride), segment after segment.
MKI_HD inline void resolve_segment_tail(uint16_t *sym, const uint8_t *hist, uint64_t o, uint64_t len, uint64_t first,
                                        uint64_t stride)
{
    const uint64_t lo = len > WSIZE ? len - WSIZE : 0;
    for (uint64_t j = lo + first; j < len; j += stride)
        sym[o + j] = resolve_symbol(sym, hist, o, sym[o + j]);
}

} // namespace mki
