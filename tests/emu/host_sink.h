// TEST INFRASTRUCTURE. The host emulations' TableSink (launch_tables.h): each table is copied into host memory that lives
// as long as the sink.
#pragma once
#include <cstring>
#include <vector>

#include "../../jxl_oxide_b200/csrc/launch_tables.h"

struct HostTableSink : jxlb::TableSink {
  std::vector<std::vector<uint64_t>> tables;
  const void* put(const void* src, size_t bytes) override {
    tables.emplace_back(bytes / 8 + 1);
    if (bytes) std::memcpy(tables.back().data(), src, bytes);
    return tables.back().data();
  }
};
