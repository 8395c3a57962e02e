// bb_planner.cpp — host-side fragment builder and FASTQ assembly of libbadread_b200 (no GPU involved).
//
// What the reference does per read before and after the hot path, as native multi-threaded host code:
//   * bb_planner_plan    build_fragment and friends (badread/simulate.py:91-115, 148-253, 361-387, 459-482),
//                        fragment lengths (fragment_lengths.py:47-64) and target identities (identities.py:76-94).
//                        Output: fragment DESCRIPTORS (bb_segment runs + literal bytes) that bb_batch_upload takes as
//                        they are, the FASTQ header info and the read name.
//   * bb_fastq_format    the record assembly of simulate.py:73-86 into one caller-provided buffer.
// Random streams: every read draws from its own `random.Random` and numpy `RandomState` keyed by (seed, read index)
// (badread_b200/simulate.py ReadPlanner.streams), so the read set depends on --seed only.  The samplers below are
// restated from CPython's _randommodule.c / random.py and numpy's legacy distributions (MT19937, 53-bit doubles,
// _randbelow_with_getrandbits, choices, polar gauss, Marsaglia-Tsang gamma, Johnk beta, geometric search / inversion);
// tests/test_planner.py pins this file draw for draw to the Python planner, which uses the real modules.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/badread_b200.h"

namespace {

// ------------------------------------------------------------------------------------------------ MT19937
struct MT {
    uint32_t mt[624];
    int idx;
    void init_genrand(uint32_t s) {
        mt[0] = s;
        for (int i = 1; i < 624; i++) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
        idx = 624;
    }
    void init_by_array(const uint32_t *key, int klen) {
        init_genrand(19650218u);
        int i = 1, j = 0;
        for (int k = (624 > klen ? 624 : klen); k; k--) {
            mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
            i++; j++;
            if (i >= 624) { mt[0] = mt[623]; i = 1; }
            if (j >= klen) j = 0;
        }
        for (int k = 623; k; k--) {
            mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
            i++;
            if (i >= 624) { mt[0] = mt[623]; i = 1; }
        }
        mt[0] = 0x80000000u;
        idx = 624;
    }
    uint32_t next() {
        if (idx >= 624) {
            for (int k = 0; k < 624; k++) {
                const uint32_t y = (mt[k] & 0x80000000u) | (mt[(k + 1) % 624] & 0x7fffffffu);
                mt[k] = mt[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            }
            idx = 0;
        }
        uint32_t y = mt[idx++];
        y ^= y >> 11;
        y ^= (y << 7) & 0x9d2c5680u;
        y ^= (y << 15) & 0xefc60000u;
        y ^= y >> 18;
        return y;
    }
    double next_double() {
        const uint32_t a = next() >> 5, b = next() >> 6;
        return (a * 67108864.0 + b) / 9007199254740992.0;
    }
};

// ------------------------------------------------------------------------------------------------ random.Random
struct PyRandom {
    MT g;
    // random.Random(x) for a non-negative int x < 2^128 given as four little-endian 32-bit words
    void seed_words(const uint32_t w[4]) {
        int n = 4;
        while (n > 1 && w[n - 1] == 0) n--;
        g.init_by_array(w, n);
    }
    double random() { return g.next_double(); }
    uint64_t getrandbits(int k) {  // 1 <= k <= 64
        if (k <= 32) return g.next() >> (32 - k);
        const uint64_t lo = g.next();
        const uint64_t hi = g.next() >> (64 - k);
        return lo | (hi << 32);
    }
    uint64_t randbelow(uint64_t n) {  // Random._randbelow_with_getrandbits
        int k = 0;
        for (uint64_t v = n; v; v >>= 1) k++;
        uint64_t r = getrandbits(k);
        while (r >= n) r = getrandbits(k);
        return r;
    }
    int64_t randint(int64_t a, int64_t b) { return a + (int64_t)randbelow((uint64_t)(b - a + 1)); }
};

// ------------------------------------------------------------------------------------------------ numpy RandomState
struct NpLegacy {
    MT g;
    bool has_gauss = false;
    double gauss_v = 0.0;
    void seed_array(const uint32_t *key, int n) { g.init_by_array(key, n); has_gauss = false; gauss_v = 0.0; }
    double dbl() { return g.next_double(); }
    double gauss() {
        if (has_gauss) { const double t = gauss_v; has_gauss = false; gauss_v = 0.0; return t; }
        double f, x1, x2, r2;
        do {
            x1 = 2.0 * dbl() - 1.0;
            x2 = 2.0 * dbl() - 1.0;
            r2 = x1 * x1 + x2 * x2;
        } while (r2 >= 1.0 || r2 == 0.0);
        f = std::sqrt(-2.0 * std::log(r2) / r2);
        gauss_v = f * x1;
        has_gauss = true;
        return f * x2;
    }
    double std_exponential() { return -std::log(1.0 - dbl()); }
    double std_gamma(double shape) {
        if (shape == 1.0) return std_exponential();
        if (shape == 0.0) return 0.0;
        if (shape < 1.0) {
            for (;;) {
                const double U = dbl();
                const double V = std_exponential();
                if (U <= 1.0 - shape) {
                    const double X = std::pow(U, 1. / shape);
                    if (X <= V) return X;
                } else {
                    const double Y = -std::log((1 - U) / shape);
                    const double X = std::pow(1.0 - shape + shape * Y, 1. / shape);
                    if (X <= (V + Y)) return X;
                }
            }
        }
        const double b = shape - 1. / 3.;
        const double c = 1. / std::sqrt(9 * b);
        for (;;) {
            double X, V;
            do {
                X = gauss();
                V = 1.0 + c * X;
            } while (V <= 0.0);
            V = V * V * V;
            const double U = dbl();
            if (U < 1.0 - 0.0331 * (X * X) * (X * X)) return b * V;
            if (std::log(U) < 0.5 * X * X + b * (1. - V + std::log(V))) return b * V;
        }
    }
    double gamma(double shape, double scale) { return scale * std_gamma(shape); }
    double beta(double a, double b) {
        if (a <= 1.0 && b <= 1.0) {
            for (;;) {  // Johnk's algorithm
                const double U = dbl(), V = dbl();
                const double X = std::pow(U, 1.0 / a), Y = std::pow(V, 1.0 / b);
                const double XpY = X + Y;
                if (XpY <= 1.0 && U + V > 0.0) {
                    if (XpY > 0) return X / XpY;
                    double logX = std::log(U) / a, logY = std::log(V) / b;
                    const double logM = logX > logY ? logX : logY;
                    logX -= logM; logY -= logM;
                    return std::exp(logX - std::log(std::exp(logX) + std::exp(logY)));
                }
            }
        }
        const double Ga = std_gamma(a), Gb = std_gamma(b);
        return Ga / (Ga + Gb);
    }
    int64_t geometric(double p) {
        if (p >= 0.333333333333333333333333) {
            int64_t X = 1;
            double sum = p, prod = p;
            const double q = 1.0 - p;
            const double U = dbl();
            while (U > sum) { prod *= q; sum += prod; X++; }
            return X;
        }
        return (int64_t)std::ceil(std::log(1.0 - dbl()) / std::log(1.0 - p));
    }
    double normal(double loc, double scale) { return loc + scale * gauss(); }
    uint8_t base() { return (uint8_t)"ACGT"[g.next() & 3u]; }  // randint(0, 4): one 32-bit word, masked
};

// ------------------------------------------------------------------------------------------------ planner
struct Piece {  // one run of a fragment: reference slice on a strand (coordinates of that strand) or literal bytes
    int32_t contig;   // -1: literal
    int32_t strand;   // 0 '+', 1 '-'
    int64_t start;    // ref: start on that strand; literal: offset into the read's literal scratch
    int64_t length;
};

struct ReadPlan {
    std::vector<Piece> pieces;
    std::string lit;   // literal bytes of this read
    std::string info;  // ' '.join(info) of simulate.py:97-113
    double identity = 0.0;
    uint8_t name[16];
    int64_t frag_len = 0;
};

}  // namespace

struct bb_planner {
    bb_plan_config cfg;
    std::vector<int64_t> contig_off, contig_len;
    std::vector<double> cum_weights;
    std::vector<uint8_t> circular, lhp, rhp;
    std::vector<std::string> names;
    std::string start_adapter, end_adapter;
    std::string err;
    // last plan, flattened
    std::vector<uint64_t> read_index;
    std::vector<int32_t> seg_off;
    std::vector<bb_segment> segs;
    std::vector<uint8_t> literals;
    std::vector<double> identity;
    std::vector<uint8_t> read_names;
    std::vector<int64_t> info_off;
    std::string info;
    std::vector<int32_t> frag_len;
};

namespace {

struct Streams {
    PyRandom rng;
    NpLegacy nrng;
};

void make_streams(uint64_t seed, uint64_t read_index, Streams &s) {
    // random.Random((seed << 64) | (read_index << 1) | 1)
    const uint64_t lo = (read_index << 1) | 1u;
    const uint32_t w[4] = {(uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)(read_index >> 63) | (uint32_t)seed,
                           (uint32_t)(seed >> 32)};
    s.rng.seed_words(w);
    // np.random.RandomState([seed_lo, seed_hi, read_lo, read_hi, 0xB200])
    const uint32_t k[5] = {(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)read_index, (uint32_t)(read_index >> 32), 0xB200u};
    s.nrng.seed_array(k, 5);
}

inline int64_t py_round(double x) { return (int64_t)std::nearbyint(x); }  // int(round(x)): half to even

int64_t fragment_length(const bb_plan_config &c, NpLegacy &nrng) {  // fragment_lengths.py:47-64
    if (c.frag_stdev == 0) return py_round(c.frag_mean);
    const int64_t v = py_round(nrng.gamma(c.gamma_k, c.gamma_t));
    return v > 1 ? v : 1;
}

void append_literal(ReadPlan &rp, const char *data, int64_t n) {
    if (n <= 0) return;
    rp.pieces.push_back(Piece{-1, 0, (int64_t)rp.lit.size(), n});
    rp.lit.append(data, (size_t)n);
}

void random_bases(NpLegacy &nrng, int64_t n, std::string &out) {
    out.resize((size_t)(n > 0 ? n : 0));
    for (int64_t i = 0; i < n; i++) out[(size_t)i] = (char)nrng.base();
}

int64_t adapter_frag_length(double amount, int64_t adapter_len, NpLegacy &nrng) {  // simulate.py:390-394
    const double beta_a = 2.0 * amount;
    const double beta_b = 2.0 - beta_a;
    return (int64_t)((double)adapter_len * nrng.beta(beta_a, beta_b));  // round(int(x)) == int(x)
}

// get_real_fragment (simulate.py:183-246): false = "return [], ''" (the caller tries again)
bool real_fragment(const bb_planner &P, int64_t fragment_length, PyRandom &rng, ReadPlan &rp, std::string &info) {
    const int n = (int)P.contig_len.size();
    int c = 0;
    if (n > 1) {  // random.choices(contigs, weights)[0]
        const double total = P.cum_weights[(size_t)n - 1] + 0.0;
        const double x = rng.random() * total;
        int lo = 0, hi = n - 1;
        while (lo < hi) {
            const int mid = (lo + hi) / 2;
            if (x < P.cum_weights[(size_t)mid]) hi = mid; else lo = mid + 1;
        }
        c = lo;
    }
    const int64_t length = P.contig_len[(size_t)c];
    const int strand = rng.random() < 0.5 ? 0 : 1;
    info = P.names[(size_t)c];
    info += strand == 0 ? ",+strand" : ",-strand";
    const bool hairpin_at_end = strand == 0 ? P.rhp[(size_t)c] : P.lhp[(size_t)c];
    char buf[96];
    if (fragment_length >= length && !P.circular[(size_t)c] && !hairpin_at_end) {
        std::snprintf(buf, sizeof(buf), ",0-%lld", (long long)length);
        info += buf;
        rp.pieces.push_back(Piece{c, strand, 0, length});
        return true;
    }
    if (fragment_length > length && P.circular[(size_t)c]) return false;
    const int64_t start_pos = rng.randint(0, length - 1);
    int64_t end_pos = start_pos + fragment_length;
    if (P.circular[(size_t)c]) {
        std::snprintf(buf, sizeof(buf), ",%lld-%lld", (long long)start_pos, (long long)end_pos);
        info += buf;
        if (end_pos <= length) { rp.pieces.push_back(Piece{c, strand, start_pos, end_pos - start_pos}); return true; }
        rp.pieces.push_back(Piece{c, strand, start_pos, length - start_pos});
        rp.pieces.push_back(Piece{c, strand, 0, end_pos - length});
        return true;
    }
    if (end_pos > length) {
        if (hairpin_at_end) {
            const int64_t fwd_len = length - start_pos;
            const int64_t left_over = std::min(fragment_length - fwd_len, fwd_len);
            std::snprintf(buf, sizeof(buf), ",%lld-%lld (hairpin) 0-%lld", (long long)start_pos, (long long)length,
                          (long long)left_over);
            info += buf;
            rp.pieces.push_back(Piece{c, strand, start_pos, fwd_len});
            rp.pieces.push_back(Piece{c, 1 - strand, 0, left_over});
            return true;
        }
        end_pos = length;
    }
    std::snprintf(buf, sizeof(buf), ",%lld-%lld", (long long)start_pos, (long long)end_pos);
    info += buf;
    rp.pieces.push_back(Piece{c, strand, start_pos, end_pos - start_pos});
    return true;
}

// get_fragment (simulate.py:148-165, 168-180, 249-253); false: 1000 failed attempts (the reference exits)
bool get_fragment(const bb_planner &P, Streams &s, ReadPlan &rp, std::string &info) {
    const bb_plan_config &c = P.cfg;
    const int64_t flen = fragment_length(c, s.nrng);
    const double draw = s.rng.random();
    std::string tmp;
    if (draw < c.junk_rate) {
        const int64_t repeat_length = s.rng.randint(1, 5);
        const int64_t repeat_count = py_round((double)flen / (double)repeat_length) + 1;
        random_bases(s.nrng, repeat_length, tmp);
        std::string junk;
        junk.reserve((size_t)(repeat_length * repeat_count));
        for (int64_t i = 0; i < repeat_count; i++) junk += tmp;
        if ((int64_t)junk.size() > flen) junk.resize((size_t)flen);
        append_literal(rp, junk.data(), (int64_t)junk.size());
        info = "junk_seq";
        return true;
    }
    if (draw < c.junk_rate + c.random_rate) {
        random_bases(s.nrng, flen, tmp);
        append_literal(rp, tmp.data(), flen);
        info = "random_seq";
        return true;
    }
    for (int attempt = 0; attempt < 1000; attempt++)
        if (real_fragment(P, flen, s.rng, rp, info)) return true;
    return false;
}

// slice_pieces(pieces, lo, hi) appended to out
void slice_into(const std::vector<Piece> &pieces, int64_t lo, int64_t hi, std::vector<Piece> &out) {
    int64_t pos = 0;
    for (const Piece &p : pieces) {
        const int64_t a = std::max(lo, pos), b = std::min(hi, pos + p.length);
        if (a < b) out.push_back(Piece{p.contig, p.strand, p.start + (a - pos), b - a});
        pos += p.length;
        if (pos >= hi) break;
    }
}

// add_glitches (simulate.py:459-482)
void add_glitches(const bb_plan_config &c, NpLegacy &nrng, ReadPlan &rp) {
    if (c.glitch_rate == 0) return;
    int64_t total = 0;
    for (const Piece &p : rp.pieces) total += p.length;
    const double p_rate = c.glitch_rate > 1 ? 1 / c.glitch_rate : 1;
    const double p_size = c.glitch_size > 1 ? 1 / c.glitch_size : 1;
    const double p_skip = c.glitch_skip > 1 ? 1 / c.glitch_skip : 1;
    std::vector<Piece> out;
    std::string tmp;
    int64_t i = 0;
    for (;;) {
        const int64_t dist = nrng.geometric(p_rate);
        slice_into(rp.pieces, i, std::min(i + dist, total), out);
        i += dist;
        if (i >= total) break;
        if (c.glitch_size > 0) {
            const int64_t n = nrng.geometric(p_size);
            random_bases(nrng, n, tmp);
            if (n > 0) {
                out.push_back(Piece{-1, 0, (int64_t)rp.lit.size(), n});
                rp.lit.append(tmp);
            }
        }
        if (c.glitch_skip > 0) i += nrng.geometric(p_skip);
        if (i >= total) break;
    }
    rp.pieces.swap(out);
}

double get_identity(const bb_plan_config &c, NpLegacy &nrng) {  // identities.py:76-94
    for (;;) {
        double identity;
        if (c.identity_type == 0) {
            if (c.id_mean == c.id_max) identity = c.id_mean;
            else identity = c.id_max * nrng.beta(c.beta_a, c.beta_b);
        } else {
            const double qscore = nrng.normal(c.id_mean, c.id_stdev);
            identity = 1.0 - std::pow(10.0, -qscore / 10);
        }
        if (0 <= identity && identity <= 100) return identity;
    }
}

// ReadPlanner.plan (badread_b200/simulate.py) == build_fragment (simulate.py:91-115) + glitches + identity + name
bool plan_read(const bb_planner &P, uint64_t read_index, ReadPlan &rp) {
    const bb_plan_config &c = P.cfg;
    Streams s;
    make_streams(c.seed, read_index, s);
    rp.pieces.clear(); rp.lit.clear(); rp.info.clear();
    // start adapter (simulate.py:361-373)
    if (!P.start_adapter.empty() && c.start_adapter_rate != 0.0 && c.start_adapter_amount != 0.0) {
        if (s.rng.random() < c.start_adapter_rate) {
            const int64_t alen = (int64_t)P.start_adapter.size();
            if (c.start_adapter_amount == 1.0) append_literal(rp, P.start_adapter.data(), alen);
            else {
                int64_t fl = adapter_frag_length(c.start_adapter_amount, alen, s.nrng);
                fl = std::max<int64_t>(0, std::min(fl, alen));
                append_literal(rp, P.start_adapter.data() + (alen - fl), fl);
            }
        }
    }
    std::string finfo;
    if (!get_fragment(P, s, rp, finfo)) return false;
    rp.info = finfo;
    while (s.rng.random() < c.chimera_rate) {  // simulate.py:101-110
        rp.info += " chimera";
        if (s.rng.random() < c.chimera_end_adapter_chance) append_literal(rp, P.end_adapter.data(), (int64_t)P.end_adapter.size());
        if (s.rng.random() < c.chimera_start_adapter_chance) append_literal(rp, P.start_adapter.data(), (int64_t)P.start_adapter.size());
        if (!get_fragment(P, s, rp, finfo)) return false;
        rp.info += " ";
        rp.info += finfo;
    }
    // end adapter (simulate.py:376-387)
    if (!P.end_adapter.empty() && c.end_adapter_rate != 0.0 && c.end_adapter_amount != 0.0) {
        if (s.rng.random() < c.end_adapter_rate) {
            const int64_t alen = (int64_t)P.end_adapter.size();
            if (c.end_adapter_amount == 1.0) append_literal(rp, P.end_adapter.data(), alen);
            else {
                int64_t fl = adapter_frag_length(c.end_adapter_amount, alen, s.nrng);
                fl = std::max<int64_t>(0, std::min(fl, alen));
                append_literal(rp, P.end_adapter.data(), fl);
            }
        }
    }
    {   // drop empty pieces
        size_t w = 0;
        for (size_t i = 0; i < rp.pieces.size(); i++)
            if (rp.pieces[i].length > 0) rp.pieces[w++] = rp.pieces[i];
        rp.pieces.resize(w);
    }
    add_glitches(c, s.nrng, rp);
    rp.identity = get_identity(c, s.nrng);
    // uuid.UUID(int=rng.getrandbits(128)): four words, least significant first; the name prints most significant first
    uint32_t w[4];
    for (int i = 0; i < 4; i++) w[i] = s.rng.g.next();
    for (int i = 0; i < 4; i++) {
        const uint32_t v = w[3 - i];
        rp.name[4 * i] = (uint8_t)(v >> 24); rp.name[4 * i + 1] = (uint8_t)(v >> 16);
        rp.name[4 * i + 2] = (uint8_t)(v >> 8); rp.name[4 * i + 3] = (uint8_t)v;
    }
    rp.frag_len = 0;
    std::string packed;  // the literal bytes of the final pieces, in order (glitches cut and drop parts of the earlier ones)
    for (Piece &p : rp.pieces) {
        rp.frag_len += p.length;
        if (p.contig < 0) {
            const int64_t at = (int64_t)packed.size();
            packed.append(rp.lit, (size_t)p.start, (size_t)p.length);
            p.start = at;
        }
    }
    rp.lit.swap(packed);
    return true;
}

}  // namespace

extern "C" int bb_planner_create(bb_planner **out, const bb_plan_config *cfg) {
    if (!out || !cfg) return BB_ERR_ARG;
    *out = nullptr;
    if (cfg->n_contigs <= 0 || !cfg->contig_len || !cfg->contig_weight || !cfg->contig_flags || !cfg->contig_names ||
        !cfg->contig_name_off)
        return BB_ERR_ARG;
    bb_planner *P = new bb_planner();
    P->cfg = *cfg;
    const int n = cfg->n_contigs;
    int64_t off = 0;
    double run = 0.0;
    for (int i = 0; i < n; i++) {
        P->contig_off.push_back(off);
        P->contig_len.push_back(cfg->contig_len[i]);
        off += cfg->contig_len[i];
        run = i == 0 ? cfg->contig_weight[0] : run + cfg->contig_weight[i];  // list(accumulate(weights))
        P->cum_weights.push_back(run);
        P->circular.push_back((cfg->contig_flags[i] & 1) ? 1 : 0);
        P->lhp.push_back((cfg->contig_flags[i] & 2) ? 1 : 0);
        P->rhp.push_back((cfg->contig_flags[i] & 4) ? 1 : 0);
        P->names.emplace_back(cfg->contig_names + cfg->contig_name_off[i],
                              (size_t)(cfg->contig_name_off[i + 1] - cfg->contig_name_off[i]));
    }
    if (cfg->start_adapter && cfg->start_adapter_len > 0) P->start_adapter.assign((const char *)cfg->start_adapter, (size_t)cfg->start_adapter_len);
    if (cfg->end_adapter && cfg->end_adapter_len > 0) P->end_adapter.assign((const char *)cfg->end_adapter, (size_t)cfg->end_adapter_len);
    // the copies above own everything the planner reads later
    P->cfg.contig_len = nullptr; P->cfg.contig_weight = nullptr; P->cfg.contig_flags = nullptr;
    P->cfg.contig_names = nullptr; P->cfg.contig_name_off = nullptr; P->cfg.start_adapter = nullptr; P->cfg.end_adapter = nullptr;
    *out = P;
    return BB_OK;
}

extern "C" int bb_planner_destroy(bb_planner *P) {
    delete P;
    return BB_OK;
}

extern "C" const char *bb_planner_error(const bb_planner *P) { return P ? P->err.c_str() : ""; }

extern "C" int bb_planner_plan(bb_planner *P, uint64_t first_index, uint64_t stride, int32_t n_reads, int32_t n_threads) {
    if (!P || n_reads < 0 || stride == 0) return BB_ERR_ARG;
    P->err.clear();
    const int T = std::max(1, std::min<int>(n_threads, std::max(1, n_reads / 64)));
    std::vector<ReadPlan> plans((size_t)n_reads);
    std::atomic<int> next{0};
    std::atomic<int> failed{0};
    auto work = [&]() {
        for (;;) {
            const int lo = next.fetch_add(64);
            if (lo >= n_reads) break;
            const int hi = std::min(n_reads, lo + 64);
            for (int i = lo; i < hi; i++)
                if (!plan_read(*P, first_index + stride * (uint64_t)i, plans[(size_t)i])) failed.store(1);
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work);
    work();
    for (auto &t : th) t.join();
    if (failed.load()) {
        P->err = "Error: failed to generate any sequence fragments - are your read lengths incompatible with your "
                 "reference contig lengths?";
        return BB_ERR_STATE;
    }
    // flatten (ReadPlanner.add_to_batch): '-' strand slices become reverse-complement slices of the forward strand
    P->read_index.resize((size_t)n_reads); P->seg_off.assign((size_t)n_reads + 1, 0); P->identity.resize((size_t)n_reads);
    P->read_names.resize((size_t)n_reads * 16); P->info_off.assign((size_t)n_reads + 1, 0); P->frag_len.resize((size_t)n_reads);
    size_t n_seg = 0, n_lit = 0, n_info = 0;
    for (const ReadPlan &rp : plans) { n_seg += rp.pieces.size(); n_lit += rp.lit.size(); n_info += rp.info.size(); }
    if (n_seg > 0x7fffffffull) { P->err = "too many segments in one plan"; return BB_ERR_ARG; }
    P->segs.resize(n_seg); P->literals.resize(n_lit + 1); P->info.resize(n_info);
    size_t sp = 0, lp = 0, ip = 0;
    for (int i = 0; i < n_reads; i++) {
        const ReadPlan &rp = plans[(size_t)i];
        P->read_index[(size_t)i] = first_index + stride * (uint64_t)i;
        P->identity[(size_t)i] = rp.identity;
        P->frag_len[(size_t)i] = (int32_t)rp.frag_len;
        std::memcpy(&P->read_names[(size_t)i * 16], rp.name, 16);
        for (const Piece &p : rp.pieces) {
            bb_segment g;
            g.len = (int32_t)p.length;
            if (p.contig < 0) { g.kind = BB_SEG_LITERAL; g.src = (int64_t)lp + p.start; }
            else if (p.strand == 0) { g.kind = BB_SEG_REF_FWD; g.src = P->contig_off[(size_t)p.contig] + p.start; }
            else {
                g.kind = BB_SEG_REF_REV;
                g.src = P->contig_off[(size_t)p.contig] + (P->contig_len[(size_t)p.contig] - p.start - p.length);
            }
            P->segs[sp++] = g;
        }
        P->seg_off[(size_t)i + 1] = (int32_t)sp;
        std::memcpy(&P->literals[lp], rp.lit.data(), rp.lit.size());
        lp += rp.lit.size();
        std::memcpy(&P->info[ip], rp.info.data(), rp.info.size());
        ip += rp.info.size();
        P->info_off[(size_t)i + 1] = (int64_t)ip;
    }
    return BB_OK;
}

extern "C" int bb_planner_view(const bb_planner *P, bb_plan_view *v) {
    if (!P || !v) return BB_ERR_ARG;
    v->n_reads = (int32_t)P->read_index.size();
    v->read_index = P->read_index.data();
    v->seg_off = P->seg_off.data();
    v->segs = P->segs.data();
    v->literals = P->literals.data();
    v->literal_len = P->literals.empty() ? 0 : (int64_t)P->literals.size() - 1;
    v->target_identity = P->identity.data();
    v->read_names = P->read_names.data();
    v->info_off = P->info_off.data();
    v->info = P->info.data();
    v->frag_len = P->frag_len.data();
    return BB_OK;
}

// ------------------------------------------------------------------------------------------------ FASTQ
namespace {

struct Emitted { int32_t g, i; };

// simulate.py:63-70 for reads [first, n) of a finished batch dealt out over n_shards contexts (read j of the batch is read
// j / n_shards of shard j % n_shards), in read-index order: empty reads are skipped, and the loop stops once the running
// total of emitted bases reaches the target.  *next_j = the first read not consumed, *total = the running total.
int select_emitted(int32_t n_shards, const bb_plan_view *const *views, const bb_read_result *const *results, int32_t first,
                   int64_t bases_so_far, int64_t target_bases, std::vector<Emitted> &emit, int64_t *next_j, int64_t *total) {
    if (n_shards <= 0 || !views || !results || first < 0) return BB_ERR_ARG;
    int64_t n = 0;
    for (int g = 0; g < n_shards; g++) {
        if (!views[g] || !results[g]) return BB_ERR_ARG;
        n += views[g]->n_reads;
    }
    for (int g = 0; g < n_shards; g++)  // shard g must hold reads g, g + G, ...
        if (views[g]->n_reads != (n - g + n_shards - 1) / n_shards) return BB_ERR_ARG;
    int64_t sum = bases_so_far;
    int64_t j = first;
    for (; j < n && sum < target_bases; j++) {
        const int g = (int)(j % n_shards), i = (int)(j / n_shards);
        const bb_read_result &r = results[g][i];
        if (r.out_len <= 0) continue;
        emit.push_back(Emitted{g, i});
        sum += r.out_len;
    }
    *next_j = j;
    *total = sum;
    return BB_OK;
}

// The read's name: its UUID as uuid.UUID prints it (36 characters).
void append_read_name(const bb_plan_view *v, int r, std::string &h) {
    static const char hex[] = "0123456789abcdef";
    const uint8_t *nm = v->read_names + (size_t)r * 16;
    for (int b = 0; b < 16; b++) {
        if (b == 4 || b == 6 || b == 8 || b == 10) h.push_back('-');
        h.push_back(hex[nm[b] >> 4]); h.push_back(hex[nm[b] & 15]);
    }
}

// The rest of the header line after the name and a space: "{info} length={len} error-free_length={frag}
// read_identity={100*matches/columns:.3f}%" (simulate.py:73-75).
void append_read_comment(const bb_plan_view *v, int r, const bb_read_result &rr, std::string &h) {
    h.append(v->info + v->info_off[r], (size_t)(v->info_off[r + 1] - v->info_off[r]));
    const double identity = rr.columns ? (double)rr.matches / (double)rr.columns : 0.0;
    char buf[128];
    std::snprintf(buf, sizeof(buf), " length=%d error-free_length=%d read_identity=%.3f%%", rr.out_len, rr.frag_len,
                  identity * 100.0);
    h += buf;
}

}  // namespace

// simulate.py:70-86 for reads [first, n) of a finished batch, in read-index order (select_emitted): a record is
// "@{uuid} {info} length={len} error-free_length={frag} read_identity={100*matches/columns:.3f}%\n{seq}\n+\n{qual}\n".
extern "C" int bb_fastq_format_sharded(int32_t n_shards, const bb_plan_view *const *views,
                                       const bb_read_result *const *results, const uint8_t *const *seq,
                                       const uint8_t *const *qual, int32_t first, int64_t bases_so_far,
                                       int64_t target_bases, int32_t n_threads, uint8_t *out, int64_t out_cap,
                                       int64_t *out_len, int32_t *n_emitted, int64_t *bases_emitted, int32_t *next_read) {
    if (!out_len) return BB_ERR_ARG;
    std::vector<Emitted> emit;
    int64_t next_j = 0, total = 0;
    if (const int rc = select_emitted(n_shards, views, results, first, bases_so_far, target_bases, emit, &next_j, &total))
        return rc;
    std::vector<std::string> headers(emit.size());
    std::vector<int64_t> off(emit.size() + 1, 0);
    for (size_t e = 0; e < emit.size(); e++) {
        const bb_plan_view *v = views[emit[e].g];
        const int r = emit[e].i;
        const bb_read_result &rr = results[emit[e].g][r];
        std::string &h = headers[e];
        h.reserve(160);
        h.push_back('@');
        append_read_name(v, r, h);
        h.push_back(' ');
        append_read_comment(v, r, rr, h);
        h.push_back('\n');
        off[e + 1] = off[e] + (int64_t)h.size() + 2ll * rr.out_len + 4;
    }
    const int64_t need = off[emit.size()];
    *out_len = need;
    if (n_emitted) *n_emitted = (int32_t)emit.size();
    if (bases_emitted) *bases_emitted = total - bases_so_far;
    if (next_read) *next_read = (int32_t)next_j;
    if (need > out_cap || (need && (!out || !seq || !qual))) return BB_ERR_CAPACITY;
    const int T = std::max(1, std::min<int>(n_threads, (int)emit.size() / 256 + 1));
    std::atomic<size_t> next{0};
    auto work = [&]() {
        for (;;) {
            const size_t lo = next.fetch_add(128);
            if (lo >= emit.size()) break;
            const size_t hi = std::min(emit.size(), lo + 128);
            for (size_t e = lo; e < hi; e++) {
                const int g = emit[e].g;
                const bb_read_result &rr = results[g][emit[e].i];
                uint8_t *p = out + off[e];
                std::memcpy(p, headers[e].data(), headers[e].size()); p += headers[e].size();
                std::memcpy(p, seq[g] + rr.out_off, (size_t)rr.out_len); p += rr.out_len;
                *p++ = '\n'; *p++ = '+'; *p++ = '\n';
                std::memcpy(p, qual[g] + rr.out_off, (size_t)rr.out_len); p += rr.out_len;
                *p++ = '\n';
            }
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work);
    work();
    for (auto &t : th) t.join();
    return BB_OK;
}

// BAM records of the same emitted set (bb_bam_build builds them): the record sizes of bb_bam_out.cuh's bam_record_size.
extern "C" int bb_bam_layout_sharded(int32_t n_shards, const bb_plan_view *const *views, const bb_read_result *const *results,
                                     int32_t first, int64_t bases_so_far, int64_t target_bases, int64_t stream_base,
                                     int32_t *shard, int32_t *index, int64_t *stream_off, bb_bam_record *recs, int64_t *fields,
                                     uint8_t *text, int64_t text_cap, int64_t *text_len, int64_t *stream_len,
                                     int32_t *n_emitted, int64_t *bases_emitted, int32_t *next_read) {
    if (!text_len || !stream_len || stream_base < 0) return BB_ERR_ARG;
    std::vector<Emitted> emit;
    int64_t next_j = 0, total = 0;
    if (const int rc = select_emitted(n_shards, views, results, first, bases_so_far, target_bases, emit, &next_j, &total))
        return rc;
    if (!emit.empty() && (!shard || !index || !stream_off || !recs || !fields)) return BB_ERR_ARG;
    std::string all;
    all.reserve(emit.size() * 160);
    int64_t at = stream_base;
    for (size_t e = 0; e < emit.size(); e++) {
        const bb_plan_view *v = views[emit[e].g];
        const int r = emit[e].i;
        const bb_read_result &rr = results[emit[e].g][r];
        bb_bam_record &o = recs[e];
        o.out_off = rr.out_off;
        o.out_len = rr.out_len;
        o.text_off = (int64_t)all.size();
        append_read_name(v, r, all);
        o.name_len = (int32_t)((int64_t)all.size() - o.text_off);
        append_read_comment(v, r, rr, all);
        o.co_len = (int32_t)((int64_t)all.size() - o.text_off - o.name_len);
        o.reserved = 0;
        shard[e] = emit[e].g;
        index[e] = r;
        stream_off[e] = at;
        const int64_t nb = ((int64_t)rr.out_len + 1) / 2;
        const int64_t o_seq = at + 36 + o.name_len + 1;
        fields[4 * e] = o_seq;
        fields[4 * e + 1] = nb;
        fields[4 * e + 2] = o_seq + nb;
        fields[4 * e + 3] = rr.out_len;
        at = o_seq + nb + rr.out_len + 3 + o.co_len + 1;
    }
    *text_len = (int64_t)all.size();
    *stream_len = at - stream_base;
    if (n_emitted) *n_emitted = (int32_t)emit.size();
    if (bases_emitted) *bases_emitted = total - bases_so_far;
    if (next_read) *next_read = (int32_t)next_j;
    if ((int64_t)all.size() > text_cap || (!all.empty() && !text)) return BB_ERR_CAPACITY;
    if (!all.empty()) std::memcpy(text, all.data(), all.size());
    return BB_OK;
}

extern "C" int bb_fastq_format(const bb_plan_view *v,const bb_read_result *results, const uint8_t *seq, const uint8_t *qual,
                               int32_t first, int64_t bases_so_far, int64_t target_bases, int32_t n_threads, uint8_t *out,
                               int64_t out_cap, int64_t *out_len, int32_t *n_emitted, int64_t *bases_emitted,
                               int32_t *next_read) {
    return bb_fastq_format_sharded(1, &v, &results, &seq, &qual, first, bases_so_far, target_bases, n_threads, out, out_cap,
                                   out_len, n_emitted, bases_emitted, next_read);
}
