// Host-side check of csrc/size_walk.cuh (the warp-parallel size walk): the windows, the speculative lanes and the
// link repair of sw_walk_warp run here lane by lane, with the header's own sw_lane / sw_lane_start / sw_broken /
// sw_base, and the result must equal the serial walk (frame_walk's restatement, tests/test_frame_model.py `walk`).
// Every byte read is bounds-checked.  Built and driven by tests/test_size_walk.py.
#include <stdint.h>
#include "../../k4os/compression/lz4_b200/csrc/size_walk.cuh"

// The serial walk: literal runs plus matchlen + 4; -1 where the chain runs past the end.
extern "C" long long sw_serial(const uint8_t* s, long long n) {
    long long p = 0, out = 0;
    while (p < n) {
        const unsigned tok = s[p++];
        long long lit = tok >> 4;
        if (lit == 15) {
            unsigned x;
            do { if (p >= n) return -1; x = s[p++]; lit += x; } while (x == 255);
        }
        out += lit;
        p += lit;
        if (p == n) return out;
        if (p + 2 > n) return -1;
        p += 2;
        long long ml = tok & 15;
        if (ml == 15) {
            unsigned x;
            do { if (p >= n) return -1; x = s[p++]; ml += x; } while (x == 255);
        }
        out += ml + 4;
    }
    return -1;
}

// sw_walk_warp, one lane at a time.  stats: [0] windows, [1] lanes 1 .. 31 that count (before the lane that ends
// the chain), [2] those of them wrong after the speculative walk, [3] repair rounds, [4] re-walks, [5] most rounds
// in one window, [6] reads outside [0, n), [7] bytes read
extern "C" long long sw_sim(const uint8_t* s, long long n, int seg, int warm, long long* stats) {
    if (n <= 0) return -1;
    auto ld8 = [&](int64_t q) -> uint32_t {
        stats[7]++;
        if (q < 0 || q >= n) { stats[6]++; return 0; }
        return s[q];
    };
    int64_t carry = 0, acc = 0;
    for (;;) {
        stats[0]++;
        const int64_t base = k4::sw_base(carry, seg);
        int64_t a[32], b[32], start[32], lim[32], e[32], x[32], o[32];
        int st[32];
        bool walk[32];
        for (int t = 0; t < 32; t++) {
            k4::sw_lane_start(n, base, carry, t, seg, warm, &a[t], &b[t], &start[t], &lim[t]);
            e[t] = -1; x[t] = -1; o[t] = 0; st[t] = k4::SW_CUT;
            walk[t] = a[t] < n;
        }
        int live = 32;
        long long rounds = 0;
        unsigned wrong = 0;
        for (int round = 0;; round++) {
            for (int t = 0; t < 32; t++)
                if (walk[t]) {
                    st[t] = k4::sw_lane(ld8, n, start[t], a[t], b[t], lim[t], &e[t], &x[t], &o[t]);
                    if (round) stats[4]++;
                }
            int64_t px[32];
            int ps[32];
            bool bad[32];
            unsigned brk = 0;
            for (int t = 0; t < 32; t++) {          // __shfl_up_sync: lane 0 reads its own value
                px[t] = x[t ? t - 1 : 0];
                ps[t] = st[t ? t - 1 : 0];
                bad[t] = k4::sw_broken(t, e[t], st[t], px[t], ps[t]);
                brk |= (unsigned)bad[t] << t;
            }
            if (round == 0) wrong = brk;
            if (!brk) break;
            const int k = __builtin_ctz(brk);
            if (ps[k] != k4::SW_NEXT) { live = k; break; }
            rounds++;
            for (int t = 0; t < 32; t++) {
                walk[t] = bad[t] && t >= k && ps[t] == k4::SW_NEXT;
                start[t] = px[t];
                if (t == k) lim[t] = n;
            }
        }
        stats[1] += live - 1;
        stats[2] += __builtin_popcount(wrong & (live == 32 ? ~0u : (1u << live) - 1));
        stats[3] += rounds;
        if (rounds > stats[5]) stats[5] = rounds;
        for (int t = 0; t < live; t++) acc += o[t];
        const int sl = st[live - 1];
        if (sl != k4::SW_NEXT) return sl == k4::SW_END ? acc : -1;
        carry = x[31];
    }
}
