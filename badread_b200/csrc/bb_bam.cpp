// bb_bam.cpp — SAM, BAM and PAF alignment records for the model builders (include/badread_b200.h, bb_aln_parse): the fields
// of the PAF line the reference's builders would read, per mapped record, from the CIGAR, POS, FLAG and the AS:i / NM:i
// tags, plus SEQ and QUAL.  BAM arrives already inflated (bb_bgzf_decompress); records may have straddled BGZF members,
// which no longer matters here.  Host code: one pass over the records, no per-record work left to the caller.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/badread_b200.h"

#include "bb_call.h"

namespace {

// BAM's CIGAR op codes (SAM specification §4.2.2): M I D N S H P = X
constexpr char kOps[] = "MIDNSHP=X";
enum { OP_M = 0, OP_I = 1, OP_D = 2, OP_N = 3, OP_S = 4, OP_H = 5, OP_P = 6, OP_EQ = 7, OP_X = 8 };

}  // namespace

struct bb_aln_set {
    std::vector<char> ref_names, read_names;
    std::vector<int64_t> ref_name_off{0}, read_name_off{0};
    std::unordered_map<std::string, int32_t> ref_ids, read_ids;
    std::vector<int32_t> read_id, ref_id, flag, score, nm, read_len, read_start, read_end, columns;
    std::vector<int64_t> ref_start, ref_end, cigar_off{0}, seq_off{0};
    std::vector<uint32_t> cigar;
    std::vector<uint8_t> seq, qual, has_qual, full;

    int32_t ref(const char *name, size_t len) {
        std::string key(name, len);
        auto it = ref_ids.find(key);
        if (it != ref_ids.end()) return it->second;
        const int32_t id = (int32_t)ref_ids.size();
        ref_ids.emplace(key, id);
        ref_names.insert(ref_names.end(), name, name + len);
        ref_name_off.push_back((int64_t)ref_names.size());
        return id;
    }
    int32_t read(const char *name, size_t len) {
        std::string key(name, len);
        auto it = read_ids.find(key);
        if (it != read_ids.end()) return it->second;
        const int32_t id = (int32_t)read_ids.size();
        read_ids.emplace(key, id);
        read_names.insert(read_names.end(), name, name + len);
        read_name_off.push_back((int64_t)read_names.size());
        return id;
    }

    // One mapped record whose CIGAR runs (length << 4 | op) are already in `cigar` from cigar_off.back() on, and whose
    // SEQ / QUAL are in seq / qual from seq_off.back() on.
    void add(const std::string &name, int32_t rid, int32_t fl, int64_t pos, bool has_as, int32_t as, bool has_nm, int32_t nm_v,
             bool qual_present) {
        const int64_t c0 = cigar_off.back(), c1 = (int64_t)cigar.size();
        int64_t rlen = 0, qaln = 0, raln = 0, cols = 0, lead = 0, trail = 0;
        bool seen_core = false, hard = false;
        for (int64_t i = c0; i < c1; i++) {
            const uint32_t op = cigar[i] & 15u, n = cigar[i] >> 4;
            if (op == OP_N || op == OP_P)
                throw Fail{BB_ERR_ARG, "Error: the CIGAR of read " + name + " has an " + kOps[op] +
                           " operation (skipped regions and padding are not supported)"};
            if (op > OP_X) throw Fail{BB_ERR_ARG, "Error: invalid CIGAR operation in the record of read " + name};
            const bool clip = op == OP_S || op == OP_H;
            hard |= op == OP_H;
            if (op != OP_D) rlen += n;
            if (clip) {
                (seen_core ? trail : lead) += n;
            } else {
                seen_core = true;
                trail = 0;   // (a clip is trailing only if no aligned op follows it)
                if (op != OP_D) qaln += n;
                if (op != OP_I) raln += n;
                cols += n;
            }
        }
        if (!has_as) throw Fail{BB_ERR_ARG, "Error: no alignment score"};
        const bool reverse = (fl & 16) != 0;
        read_id.push_back(read(name.data(), name.size()));
        ref_id.push_back(rid);
        flag.push_back(fl);
        score.push_back(as);
        nm.push_back(has_nm ? nm_v : -1);
        read_len.push_back((int32_t)rlen);
        read_start.push_back((int32_t)(reverse ? trail : lead));
        read_end.push_back((int32_t)((reverse ? trail : lead) + qaln));
        columns.push_back((int32_t)cols);
        ref_start.push_back(pos);
        ref_end.push_back(pos + raln);
        cigar_off.push_back(c1);
        const bool has_seq = (int64_t)seq.size() > seq_off.back();
        has_qual.push_back(qual_present && has_seq);
        full.push_back(has_seq && !hard);
        seq_off.push_back((int64_t)seq.size());
    }
};

namespace {

bool parse_int(const char *p, const char *end, int64_t *v) {
    if (p == end) return false;
    bool neg = false;
    if (*p == '-' || *p == '+') { neg = *p == '-'; p++; }
    if (p == end) return false;
    int64_t x = 0;
    for (; p < end; p++) {
        if (*p < '0' || *p > '9') return false;
        x = x * 10 + (*p - '0');
        if (x > (int64_t)1 << 40) return false;
    }
    *v = neg ? -x : x;
    return true;
}

void parse_sam(bb_aln_set &S, const char *text, int64_t n, int64_t max_records) {
    int64_t line_no = 0, n_rec = 0;
    std::vector<std::pair<const char *, const char *>> f;
    for (const char *p = text, *end = text + n; p < end;) {
        const char *eol = (const char *)std::memchr(p, '\n', (size_t)(end - p));
        if (!eol) eol = end;
        const char *le = eol > p && eol[-1] == '\r' ? eol - 1 : eol;
        line_no++;
        const char *line = p;
        p = eol + 1;
        if (le == line) continue;
        f.clear();
        for (const char *q = line;;) {
            const char *tab = (const char *)std::memchr(q, '\t', (size_t)(le - q));
            f.emplace_back(q, tab ? tab : le);
            if (!tab) break;
            q = tab + 1;
        }
        if (*line == '@') {   // header: reference names of @SQ lines, in order
            if (le - line >= 3 && std::memcmp(line, "@SQ", 3) == 0)
                for (auto &x : f)
                    if (x.second - x.first > 3 && std::memcmp(x.first, "SN:", 3) == 0) S.ref(x.first + 3, (size_t)(x.second - x.first - 3));
            continue;
        }
        int64_t fl = 0, pos = 0;
        if (f.size() < 11 || !parse_int(f[1].first, f[1].second, &fl) || !parse_int(f[3].first, f[3].second, &pos)) {
            char msg[128];
            std::snprintf(msg, sizeof(msg), "Error: line %lld of the alignment file is not a SAM record", (long long)line_no);
            throw Fail{BB_ERR_ARG, msg};
        }
        const std::string rname(f[2].first, f[2].second);
        if ((fl & 4) || rname == "*") continue;
        const std::string name(f[0].first, f[0].second);
        if (f[5].second - f[5].first == 1 && *f[5].first == '*') throw Fail{BB_ERR_ARG, "Error: no CIGAR string found"};
        for (const char *c = f[5].first; c < f[5].second;) {
            int64_t len = 0;
            const char *d = c;
            while (d < f[5].second && *d >= '0' && *d <= '9' && len < ((int64_t)1 << 28)) len = len * 10 + (*d++ - '0');
            const char *op = d < f[5].second ? std::strchr(kOps, *d) : nullptr;
            if (d == c || !op || !*d) throw Fail{BB_ERR_ARG, "Error: invalid CIGAR string in the record of read " + name};
            S.cigar.push_back(((uint32_t)len << 4) | (uint32_t)(op - kOps));
            c = d + 1;
        }
        const bool has_seq = !(f[9].second - f[9].first == 1 && *f[9].first == '*');
        const bool has_qual = !(f[10].second - f[10].first == 1 && *f[10].first == '*');
        if (has_seq) {
            for (const char *c = f[9].first; c < f[9].second; c++) S.seq.push_back((uint8_t)(*c >= 'a' && *c <= 'z' ? *c - 32 : *c));
            const int64_t ns = f[9].second - f[9].first;
            for (int64_t i = 0; i < ns; i++)
                S.qual.push_back(has_qual && i < f[10].second - f[10].first ? (uint8_t)f[10].first[i] : (uint8_t)0);
        }
        bool has_as = false, has_nm = false;
        int64_t as = 0, nm = 0;
        for (size_t k = 11; k < f.size(); k++) {
            const char *t = f[k].first, *te = f[k].second;
            if (te - t > 5 && t[2] == ':' && t[3] == 'i' && t[4] == ':') {
                if (t[0] == 'A' && t[1] == 'S' && !has_as) has_as = parse_int(t + 5, te, &as);
                if (t[0] == 'N' && t[1] == 'M' && !has_nm) has_nm = parse_int(t + 5, te, &nm);
            }
        }
        S.add(name, S.ref(rname.data(), rname.size()), (int32_t)fl, pos - 1, has_as, (int32_t)as, has_nm, (int32_t)nm, has_qual);
        if (++n_rec == max_records) break;
    }
}

void parse_bam(bb_aln_set &S, const uint8_t *d, int64_t n, int64_t max_records) {
    auto need = [&](int64_t at, int64_t len, const char *what) {
        if (at < 0 || len < 0 || at + len > n) throw Fail{BB_ERR_ARG, std::string("Error: the BAM file is truncated (") + what + ")"};
    };
    auto i32 = [&](int64_t at) { int32_t v; std::memcpy(&v, d + at, 4); return v; };
    auto u16 = [&](int64_t at) { uint16_t v; std::memcpy(&v, d + at, 2); return v; };
    need(0, 12, "header");
    if (std::memcmp(d, "BAM\1", 4) != 0) throw Fail{BB_ERR_ARG, "Error: the alignment file is not BAM (no BAM magic after inflating)"};
    int64_t at = 8 + (int64_t)i32(4);
    need(at, 4, "header");
    const int32_t n_ref = i32(at);
    at += 4;
    if (n_ref < 0) throw Fail{BB_ERR_ARG, "Error: the BAM header is invalid (negative reference count)"};
    for (int32_t r = 0; r < n_ref; r++) {
        need(at, 4, "reference names");
        const int32_t l_name = i32(at);
        need(at + 4, (int64_t)l_name + 4, "reference names");
        if (l_name < 1) throw Fail{BB_ERR_ARG, "Error: the BAM header is invalid (empty reference name)"};
        if (S.ref((const char *)d + at + 4, (size_t)l_name - 1) != r) throw Fail{BB_ERR_ARG, "Error: the BAM header names a reference twice"};
        at += 4 + (int64_t)l_name + 4;
    }
    int64_t n_rec = 0;
    static const char kSeq[] = "=ACMGRSVTWYHKDBN";
    while (at < n) {
        need(at, 4, "record");
        const int64_t bs = i32(at), r0 = at + 4, r1 = r0 + bs;
        need(r0, bs, "record");
        if (bs < 32) throw Fail{BB_ERR_ARG, "Error: the BAM file holds an invalid record"};
        at = r1;
        const int32_t ref_id = i32(r0), pos = i32(r0 + 4);
        const int l_name = d[r0 + 8];
        const int n_cig = u16(r0 + 12), fl = u16(r0 + 14);
        const int32_t l_seq = i32(r0 + 16);
        const int64_t p_name = r0 + 32, p_cig = p_name + l_name, p_seq = p_cig + 4 * (int64_t)n_cig;
        const int64_t p_qual = p_seq + ((int64_t)l_seq + 1) / 2, p_tags = p_qual + l_seq;
        if (l_name < 1 || l_seq < 0 || p_tags > r1) throw Fail{BB_ERR_ARG, "Error: the BAM file holds an invalid record"};
        if ((fl & 4) || ref_id < 0) continue;
        if (ref_id >= n_ref) throw Fail{BB_ERR_ARG, "Error: a BAM record names a reference the header does not list"};
        const std::string name((const char *)d + p_name, (size_t)l_name - 1);
        if (n_cig == 0) throw Fail{BB_ERR_ARG, "Error: no CIGAR string found"};
        for (int k = 0; k < n_cig; k++) {
            uint32_t c;
            std::memcpy(&c, d + p_cig + 4 * k, 4);
            S.cigar.push_back(c);
        }
        const bool has_qual = l_seq > 0 && d[p_qual] != 0xff;
        for (int32_t i = 0; i < l_seq; i++) {
            S.seq.push_back((uint8_t)kSeq[(d[p_seq + i / 2] >> (i & 1 ? 0 : 4)) & 15]);
            S.qual.push_back(has_qual ? (uint8_t)(d[p_qual + i] + 33) : (uint8_t)0);
        }
        bool has_as = false, has_nm = false;
        int64_t as = 0, nm = 0;
        for (int64_t t = p_tags; t < r1;) {
            need(t, 3, "tags");
            if (t + 3 > r1) throw Fail{BB_ERR_ARG, "Error: the BAM file holds an invalid record"};
            const char a = (char)d[t], b = (char)d[t + 1], type = (char)d[t + 2];
            int64_t v = 0, size;
            t += 3;
            switch (type) {
                case 'A': case 'c': case 'C': size = 1; break;
                case 's': case 'S': size = 2; break;
                case 'i': case 'I': case 'f': size = 4; break;
                case 'Z': case 'H': {
                    const void *z = t < r1 ? std::memchr(d + t, 0, (size_t)(r1 - t)) : nullptr;
                    if (!z) throw Fail{BB_ERR_ARG, "Error: the BAM file holds an invalid record"};
                    size = (const uint8_t *)z - (d + t) + 1;
                    break;
                }
                case 'B': {
                    if (t + 5 > r1) throw Fail{BB_ERR_ARG, "Error: the BAM file holds an invalid record"};
                    const char sub = (char)d[t];
                    const int64_t w = sub == 'c' || sub == 'C' ? 1 : sub == 's' || sub == 'S' ? 2 : 4;
                    size = 5 + w * (int64_t)(uint32_t)i32(t + 1);
                    break;
                }
                default: throw Fail{BB_ERR_ARG, "Error: the BAM file holds an invalid record"};
            }
            if (t + size > r1) throw Fail{BB_ERR_ARG, "Error: the BAM file holds an invalid record"};
            const bool integer = type == 'c' || type == 'C' || type == 's' || type == 'S' || type == 'i' || type == 'I';
            if (integer) {
                switch (type) {
                    case 'c': v = (int8_t)d[t]; break;
                    case 'C': v = d[t]; break;
                    case 's': v = (int16_t)u16(t); break;
                    case 'S': v = u16(t); break;
                    case 'i': v = i32(t); break;
                    default: v = (uint32_t)i32(t); break;
                }
                if (a == 'A' && b == 'S' && !has_as) { has_as = true; as = v; }
                if (a == 'N' && b == 'M' && !has_nm) { has_nm = true; nm = v; }
            }
            t += size;
        }
        S.add(name, ref_id, fl, pos, has_as, (int32_t)as, has_nm, (int32_t)nm, has_qual);
        if (++n_rec == max_records) break;
    }
}

// str.strip()'s ASCII whitespace
bool paf_space(char c) { return c == ' ' || (c >= '\t' && c <= '\r') || (c >= 0x1c && c <= 0x1f); }

// PAF text as model_builders.Alignment reads it, line by line (text mode: '\n', "\r\n" and a lone '\r' end lines)
void parse_paf(bb_aln_set &S, const char *text, int64_t n, int64_t max_records) {
    int64_t line_no = 0;
    std::vector<std::pair<const char *, const char *>> f;
    for (const char *p = text, *end = text + n; p < end;) {
        const char *q = p;
        while (q < end && *q != '\n' && *q != '\r') q++;
        const char *line = p, *le = q;
        p = q == end ? end : (*q == '\r' && q + 1 < end && q[1] == '\n') ? q + 2 : q + 1;
        line_no++;
        while (line < le && paf_space(*line)) line++;
        while (le > line && paf_space(le[-1])) le--;
        f.clear();
        for (const char *c = line;;) {
            const char *tab = (const char *)std::memchr(c, '\t', (size_t)(le - c));
            f.emplace_back(c, tab ? tab : le);
            if (!tab) break;
            c = tab + 1;
        }
        if (f.size() < 11) throw Fail{BB_ERR_ARG, "Error: alignment file does not seem to be in PAF format"};
        // int() of a field: surrounding whitespace, an optional sign, decimal digits
        auto num = [&](const char *a, const char *b, int64_t lo, int64_t hi, const char *what) {
            while (a < b && paf_space(*a)) a++;
            while (b > a && paf_space(b[-1])) b--;
            int64_t v = 0;
            if (!parse_int(a, b, &v) || v < lo || v > hi) {
                char msg[160];
                std::snprintf(msg, sizeof(msg), "Error: %s on line %lld of the alignment file is not an integer in [%lld, %lld]",
                              what, (long long)line_no, (long long)lo, (long long)hi);
                throw Fail{BB_ERR_ARG, msg};
            }
            return v;
        };
        auto col = [&](int k, int64_t lo, int64_t hi) {
            static const char *names[] = {"", "", "column 3", "column 4", "", "", "", "column 8", "column 9", "column 10", "column 11"};
            return num(f[k].first, f[k].second, lo, hi, names[k]);
        };
        const int64_t qs = col(2, INT32_MIN, INT32_MAX), qe = col(3, INT32_MIN, INT32_MAX);
        const int64_t ts = col(7, -((int64_t)1 << 40), (int64_t)1 << 40), te = col(8, -((int64_t)1 << 40), (int64_t)1 << 40);
        const int64_t matching = col(9, INT32_MIN, INT32_MAX), cols = col(10, INT32_MIN, INT32_MAX);
        if (cols == 0) {
            char msg[128];
            std::snprintf(msg, sizeof(msg), "Error: line %lld of the alignment file has 0 alignment columns (column 11)", (long long)line_no);
            throw Fail{BB_ERR_ARG, msg};
        }
        if (cols - matching < INT32_MIN || cols - matching > INT32_MAX) {
            char msg[128];
            std::snprintf(msg, sizeof(msg), "Error: columns 10 and 11 on line %lld of the alignment file are out of range", (long long)line_no);
            throw Fail{BB_ERR_ARG, msg};
        }
        const char *cg = nullptr, *cg_end = nullptr;
        bool has_as = false;
        int64_t as = 0;
        for (auto &x : f) {   // every column, the last tag of each kind wins
            if (x.second - x.first >= 5 && std::memcmp(x.first, "cg:Z:", 5) == 0) { cg = x.first + 5; cg_end = x.second; }
            if (x.second - x.first >= 5 && std::memcmp(x.first, "AS:i:", 5) == 0) {
                as = num(x.first + 5, x.second, INT32_MIN, INT32_MAX, "the AS:i: tag");
                has_as = true;
            }
        }
        if (!cg) throw Fail{BB_ERR_ARG, "Error: no CIGAR string found"};
        if (!has_as) throw Fail{BB_ERR_ARG, "Error: no alignment score"};
        const std::string name(f[0].first, f[0].second);
        for (const char *c = cg; c < cg_end;) {   // re.findall(r'(\d+)([A-Za-z=])')
            if (*c < '0' || *c > '9') { c++; continue; }
            const char *d = c;
            while (d < cg_end && *d >= '0' && *d <= '9') d++;
            const bool letter = d < cg_end && ((*d >= 'A' && *d <= 'Z') || (*d >= 'a' && *d <= 'z') || *d == '=');
            if (!letter) { c = d; continue; }
            const uint32_t code = *d == 'M' ? OP_M : *d == 'I' ? OP_I : *d == 'D' ? OP_D : 15u;
            int64_t len = 0;
            for (const char *x = c; x < d && len < ((int64_t)1 << 28); x++) len = len * 10 + (*x - '0');
            if (code != 15u && len >= ((int64_t)1 << 28)) throw Fail{BB_ERR_ARG, "Error: a CIGAR run of read " + name + " is longer than 2^28 - 1"};
            S.cigar.push_back(((uint32_t)(code == 15u ? 0 : len) << 4) | code);
            c = d + 1;
        }
        const bool reverse = f[4].second - f[4].first == 1 && *f[4].first == '-';
        S.read_id.push_back(S.read(name.data(), name.size()));
        S.ref_id.push_back(S.ref(f[5].first, (size_t)(f[5].second - f[5].first)));
        S.flag.push_back(reverse ? 16 : 0);
        S.score.push_back((int32_t)as);
        S.nm.push_back((int32_t)(cols - matching));
        S.read_len.push_back(0);
        S.read_start.push_back((int32_t)qs);
        S.read_end.push_back((int32_t)qe);
        S.columns.push_back((int32_t)cols);
        S.ref_start.push_back(ts);
        S.ref_end.push_back(te);
        S.cigar_off.push_back((int64_t)S.cigar.size());
        S.has_qual.push_back(0);
        S.full.push_back(0);
        S.seq_off.push_back((int64_t)S.seq.size());
        if (line_no == max_records) break;
    }
}

}  // namespace

extern "C" int bb_aln_parse(const uint8_t *data, int64_t n, int is_bam, int64_t max_records, bb_aln_set **set) {
    if (!set || n < 0 || (n > 0 && !data)) return bad_argument("bb_aln_parse");
    *set = nullptr;
    return model_call([&] {
        std::unique_ptr<bb_aln_set> S(new bb_aln_set());
        if (is_bam == BB_ALN_PAF) parse_paf(*S, (const char *)data, n, max_records);
        else if (is_bam) parse_bam(*S, data, n, max_records);
        else parse_sam(*S, (const char *)data, n, max_records);
        *set = S.release();
        return BB_OK;
    });
}

extern "C" int bb_aln_view_get(const bb_aln_set *S, bb_aln_view *v) {
    if (!S || !v) return BB_ERR_ARG;
    v->n_records = (int64_t)S->read_id.size();
    v->n_refs = (int32_t)(S->ref_name_off.size() - 1);
    v->n_reads = (int32_t)(S->read_name_off.size() - 1);
    v->ref_names = S->ref_names.data();
    v->ref_name_off = S->ref_name_off.data();
    v->read_names = S->read_names.data();
    v->read_name_off = S->read_name_off.data();
    v->read_id = S->read_id.data();
    v->ref_id = S->ref_id.data();
    v->flag = S->flag.data();
    v->score = S->score.data();
    v->nm = S->nm.data();
    v->read_len = S->read_len.data();
    v->read_start = S->read_start.data();
    v->read_end = S->read_end.data();
    v->columns = S->columns.data();
    v->ref_start = S->ref_start.data();
    v->ref_end = S->ref_end.data();
    v->cigar = S->cigar.data();
    v->cigar_off = S->cigar_off.data();
    v->seq = S->seq.data();
    v->qual = S->qual.data();
    v->seq_off = S->seq_off.data();
    v->has_qual = S->has_qual.data();
    v->full = S->full.data();
    return BB_OK;
}

extern "C" int bb_aln_free(bb_aln_set *S) {
    delete S;
    return BB_OK;
}
