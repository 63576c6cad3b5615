// block_combine_bench.cpp — the YQL single-key BlockCombineHashed shape, two ways: the existing adapter
// (CreateGpuBlockCombineHashed: per-batch GPU GROUP BY, partial states merged on the host at Finish) against the GROUP BY
// table adapter (CreateGpuBlockCombineHashedKeys), over the same Arrow batches of an int64 key and an int64 value with
// SUM and COUNT.  Run by bench_groupby_table.py; prints one JSON line: per group count, the wall time of all AddBlock
// calls plus Finish for each adapter (median of `steps` after one warm-up), and whether their groups, sums and counts
// agree.  Usage: block_combine_bench ROWS BATCH STEPS
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <random>
#include <vector>

#include "../../include/ytgpu.h"
#include "../yt_query_client.h"

using namespace NYql::NMiniKQL;
using namespace NYT::NQueryClient;

namespace {

TArrowColumn Col(const std::vector<uint64_t>& v, int64_t from, int64_t n) {
    TArrowColumn a;
    a.Values = v.data();
    a.Offset = from;
    a.Length = n;
    a.ValueType = YTGPU_TYPE_INT64;
    return a;
}

double Seconds(std::chrono::steady_clock::time_point a) {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - a).count();
}

}  // namespace

int main(int argc, char** argv) {
    const int64_t rows = argc > 1 ? std::atoll(argv[1]) : (1ll << 26);
    const int64_t batch = argc > 2 ? std::atoll(argv[2]) : (1ll << 20);
    const int steps = argc > 3 ? std::atoi(argv[3]) : 3;
    std::printf("{\"rows\": %lld, \"batch\": %lld, \"legs\": {", (long long)rows, (long long)batch);
    bool firstLeg = true;
    for (uint64_t groups : {1000ull, 1000000ull}) {
        std::mt19937_64 rng(groups);
        std::vector<uint64_t> key(rows), value(rows);
        for (int64_t i = 0; i < rows; ++i) {
            key[i] = rng() % groups;
            value[i] = (uint64_t)((int64_t)(rng() % 2000001) - 1000000);
        }
        std::vector<double> partial, table;
        IBlockCombineHashed::TResult a;
        IBlockCombineHashedKeys::TResult b;
        for (int s = 0; s <= steps; ++s) {
            auto t0 = std::chrono::steady_clock::now();
            auto p = CreateGpuBlockCombineHashed(groups);
            for (int64_t i = 0; i < rows; i += batch) p->AddBlock(Col(key, i, std::min(batch, rows - i)), Col(value, i, std::min(batch, rows - i)));
            a = p->Finish();
            if (s) partial.push_back(Seconds(t0));
            t0 = std::chrono::steady_clock::now();
            auto t = CreateGpuBlockCombineHashedKeys({{EAggregateFunction::Sum, 0, -1}, {EAggregateFunction::Count, 0, -1}}, groups);
            for (int64_t i = 0; i < rows; i += batch) t->AddBlock({Col(key, i, std::min(batch, rows - i))}, {Col(value, i, std::min(batch, rows - i))});
            b = t->Finish();
            if (s) table.push_back(Seconds(t0));
        }
        // parity: the same groups with the same sums and counts (the partial-state adapter's order is its own)
        std::map<uint64_t, std::pair<uint64_t, uint64_t>> ra, rb;
        for (size_t i = 0; i < a.Keys.size(); ++i) ra[a.Keys[i]] = {a.Sums[i], a.Counts[i]};
        for (size_t i = 0; i < b.Keys[0].size(); ++i) rb[b.Keys[0][i]] = {b.Values[0][i], b.Values[1][i]};
        std::sort(partial.begin(), partial.end());
        std::sort(table.begin(), table.end());
        std::printf("%s\"yql_single_key_%llu\": {\"partial_states_ms\": %.3f, \"table_ms\": %.3f, \"parity\": %s}", firstLeg ? "" : ", ",
                    (unsigned long long)groups, 1e3 * partial[partial.size() / 2], 1e3 * table[table.size() / 2], ra == rb ? "true" : "false");
        firstLeg = false;
    }
    std::printf("}}\n");
    return 0;
}
