// Host-side check of csrc/parse_table.cuh (the decoder's jump table): every table byte that is not the
// escape value must equal the distance to the next token that a strict restatement of the LZ4 block
// format's length decoding gives (reference: LL64.dec.cs:191-246,300-336, LL.tools.cs:165-193), the
// sequence must be neither terminal nor malformed, and jt_outbytes must equal its decoded size.
// Built and driven by tests/test_parse_table.py.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../k4os/compression/lz4_b200/csrc/parse_table.cuh"

namespace {
struct Seq { int next; long outb; bool bad, last; };
Seq ref_seq(const uint8_t* s, int n, int p) {
    Seq r{n, 0, false, false};
    const unsigned tok = s[p];
    int q = p + 1;
    long lit = tok >> 4;
    if (lit == 15) for (;;) { if (q >= n) { r.bad = true; return r; } const unsigned b = s[q++]; lit += b; if (b != 255) break; }
    const long litEnd = q + lit;
    if (litEnd + 2 > n) { r.last = true; r.outb = lit; r.bad = litEnd != n; return r; }
    long q2 = litEnd + 2, ml = tok & 15;
    if (ml == 15) for (;;) { if (q2 >= n) { r.bad = true; return r; } const unsigned b = s[q2++]; ml += b; if (b != 255) break; }
    r.next = (int)(q2 < n ? q2 : n); r.outb = lit + ml + 4; r.bad = q2 >= n;
    return r;
}
}  // namespace

// stats: [0] positions checked, [1] escapes among all positions, [2] true-chain tokens, [3] escapes among them,
// [4] first failing position + 1 (0 = none), [5] wrong lanes of a simulated speculative parse, [6] lanes
extern "C" int jt_check(const uint8_t* stream, int n, int shift, int fill, int seg, int warm, long long* stats) {
    std::vector<uint8_t> stage((size_t)shift + n + 64, (uint8_t)fill);
    if (fill > 255) {        // pseudo-random bytes seeded by `fill`: the big-stage kernel sees the previous block's bytes
        uint32_t x = (uint32_t)fill * 2654435761u;
        for (auto& b : stage) { x = x * 1664525u + 1013904223u; b = (uint8_t)(x >> 24); }
    }
    memcpy(stage.data() + shift, stream, (size_t)n);
    const uint8_t* s = stage.data() + shift;                 // s[p] = stream byte p; bytes at >= n (and < 0) are `fill`
    std::vector<uint8_t> J((size_t)shift + n + 64, 0);
    auto ld8 = [&](int q) -> uint32_t { return s[q]; };
    const int nWords = (shift + n + 3) >> 2;
    for (int k = 0; k < nWords; k++) {
        uint32_t w0, w1;
        memcpy(&w0, stage.data() + 4 * k, 4); memcpy(&w1, stage.data() + 4 * k + 4, 4);
        const uint32_t out = k4::jt_word(w0, w1, 4 * k - shift, n, ld8);
        memcpy(J.data() + 4 * k, &out, 4);
    }
    const uint8_t* Jp = J.data() + shift;
    int fails = 0;
    for (int p = 0; p < n; p++) {
        stats[0]++;
        const uint32_t j = Jp[p];
        if (j == k4::JT_ESC) { stats[1]++; continue; }
        const Seq r = ref_seq(stream, n, p);
        const bool ok = !r.bad && !r.last && r.next == p + (int)j && r.next < n &&
                        r.outb == (long)k4::jt_outbytes(p, j, ld8);
        if (!ok) { if (!fails) stats[4] = p + 1; fails++; }
    }
    // the true chain
    std::vector<int> chain;
    for (int p = 0; p < n;) {
        chain.push_back(p);
        stats[2]++;
        if (Jp[p] == k4::JT_ESC) stats[3]++;
        const Seq r = ref_seq(stream, n, p);
        if (r.bad || r.next <= p) break;
        p = r.next;
    }
    // simulated speculative parse: lane t walks from segStart - warm; wrong iff its entry is not on the true chain
    if (seg > 0) {
        std::vector<uint8_t> onChain((size_t)n + 1, 0);
        for (int p : chain) onChain[p] = 1;
        onChain[n] = 1;
        for (int t = 1; t * seg < n; t++) {
            int p = t * seg > warm ? t * seg - warm : 0;
            while (p < t * seg) { const Seq r = ref_seq(stream, n, p); if (r.next <= p) break; p = r.next; }
            stats[6]++;
            if (p >= t * seg && !onChain[p]) stats[5]++;
        }
    }
    return fails;
}
