// partitioner_golden — prints the --partitioner-check table for rows given on stdin (no GPU): used by
// tests/test_partitioner.py to pin its format to tests/golden/partitioner_report.txt.
// stdin: C, the C counts, nrows, then per row: P keyed and the 2C + 1 counters
#include <iostream>
#include "kta_report.hpp"
int main() {
    size_t c = 0, n = 0;
    std::cin >> c;
    std::vector<int32_t> counts(c);
    for (auto &v : counts) std::cin >> v;
    std::cin >> n;
    std::vector<kta_report::PartitionerRow> rows(n);
    for (auto &r : rows) {
        std::cin >> r.partition >> r.keyed;
        r.counts.resize(2 * c + 1);
        for (auto &v : r.counts) std::cin >> v;
    }
    std::cout << kta_report::render_partitioner_check(counts, rows);
}
