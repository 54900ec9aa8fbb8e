// hot_keys_golden — prints the --hot-keys report for rows given on stdin (no GPU): used by tests/test_hot_keys.py to pin its
// format to tests/golden/hot_keys_report.txt.
// stdin: distinct keys, nrows, then per row: records tombstones bytes latest_s min_partition max_partition key_len, and the
// prefix as hex ("-" when empty)
#include <iostream>
#include "kta_report.hpp"
int main() {
    uint64_t distinct = 0;
    size_t n = 0;
    std::cin >> distinct >> n;
    std::vector<kta_report::HotKeyRow> rows(n);
    for (auto &r : rows) {
        std::string hex;
        std::cin >> r.records >> r.tombstones >> r.bytes >> r.latest_s >> r.min_partition >> r.max_partition >> r.key_len >> hex;
        if (hex != "-")
            for (size_t i = 0; i + 1 < hex.size(); i += 2) r.prefix += (char)std::stoi(hex.substr(i, 2), nullptr, 16);
    }
    std::cout << kta_report::render_hot_keys(distinct, rows);
}
