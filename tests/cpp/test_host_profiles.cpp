// The C++ mirror's AlignProfiles (famsa_b200/host/famsa_b200_host.hpp) on FAMSA's profile-profile golden: argv[1] names a
// text file with the gap costs, the 24 x 24 score matrix, the two inputs (count, then one row per line) and upgma.pp.fasta's
// rows in file order.  The merged rows are rebuilt as FinalizeGaps does from the two GapRuns lists and the order, and must
// be the golden's.
#include <cstdio>
#include <fstream>
#include <iostream>

#include "../../famsa_b200/host/famsa_b200_host.hpp"

#define REQUIRE(c) do { if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

static uint8_t code(char c)
{
    static const char* letters = "ARNDCQEGHILKMFPSTWYVBZX*";
    if (c == '-') return 30;
    if (c > 'Z') c -= 32;
    for (int k = 0; k < 24; ++k)
        if (letters[k] == c) return (uint8_t)k;
    return 22;
}

// a row with the runs' gap columns inserted; the last column stays at the end (rows read as text)
static std::string finalize(const std::string& row, const std::vector<std::pair<uint32_t, uint32_t>>& runs)
{
    std::string body = row.substr(0, row.size() - 1), out;
    size_t at = 0;
    for (const auto& r : runs) {                       // run (first merged column, length), 1-based, in order
        while (out.size() + 1 < r.first) out.push_back(body[at++]);
        out.append(r.second, '-');
    }
    out.append(body, at, std::string::npos);
    return out + row.back();
}

int main(int argc, char** argv)
{
    using namespace famsa_b200;
    if (argc != 2) return 2;
    std::ifstream f(argv[1]);
    int64_t gaps[4], sm[24 * 24];
    for (auto& g : gaps) f >> g;
    for (auto& v : sm) f >> v;
    std::vector<std::string> text[2], gold;
    for (auto& t : text) {
        size_t n;
        f >> n;
        t.resize(n);
        for (auto& r : t) f >> r;
    }
    size_t ng;
    f >> ng;
    gold.resize(ng);
    for (auto& r : gold) f >> r;
    REQUIRE(f.good() && ng == text[0].size() + text[1].size());
    std::vector<std::vector<uint8_t>> rows[2];
    for (int s = 0; s < 2; ++s)
        for (auto& t : text[s]) {
            std::vector<uint8_t> r;
            for (char c : t) r.push_back(code(c));
            rows[s].push_back(r);
        }
    Context ctx(0);
    check(famsa_prof_set_scoring(ctx.get(), sm));
    const ProfileAlignment pa = AlignProfiles(ctx, rows[0], rows[1], gaps);
    REQUIRE(pa.order.size() == ng);
    const size_t n1 = text[0].size();
    for (size_t k = 0; k < ng; ++k) {
        const uint32_t i = pa.order[k];
        const std::string merged = i < n1 ? finalize(text[0][i], pa.gaps1) : finalize(text[1][i - n1], pa.gaps2);
        REQUIRE(merged == gold[k]);
    }
    uint64_t live = 0;
    check(famsa_prof_stats(ctx.get(), &live, nullptr));
    REQUIRE(live == 1);
    check(famsa_prof_drop(ctx.get(), &pa.merged_id, 1));
    bool threw = false;
    try { AlignProfiles(ctx, rows[0], {}, gaps); } catch (const std::runtime_error&) { threw = true; }
    REQUIRE(threw);
    check(famsa_prof_stats(ctx.get(), &live, nullptr));
    REQUIRE(live == 0);
    std::printf("host mirror profiles ok: %zu rows, total %lld\n", ng, (long long)pa.merge.total_score);
    return 0;
}
