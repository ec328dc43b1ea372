// Test harness (tests/test_emu_post.py): one of the three restatements of .NET's ArraySortHelper introsort, selected with -DSRC=1|2|3,
// sorts element indices by an int value with Comparison (a, b) => a.CompareTo(b). stdin: n, then n values; stdout: the sorted indices.
#include <cstdio>
#include <vector>
#include <utility>
#if SRC == 1
#define IFX_EMU 1
#include "../infidex_b200/csrc/ifx_stage1.h"          // the device's IntroSort (kernels, emulation build)
#elif SRC == 2
#include "../infidex_b200/csrc/ifx_host_build.cpp"    // the host builder's DotnetIntroSort
#else
#include "../oracle/text.hpp"                         // the oracle's DotnetSort
#endif

struct ByValue { const int* v; int operator()(int a, int b) const { return v[a] < v[b] ? -1 : (v[a] > v[b] ? 1 : 0); } };

int main() {
    int n = 0; if (scanf("%d", &n) != 1) return 1;
    std::vector<int> val(n), idx(n);
    for (int i = 0; i < n; i++) { if (scanf("%d", &val[i]) != 1) return 1; idx[i] = i; }
    ByValue by{val.data()};
#if SRC == 1
    ifx::IntroSort<ByValue> s{by}; s.sort(idx.data(), n);
#elif SRC == 2
    DotnetIntroSort<int, ByValue> s{by}; s.sort(idx.data(), n);
#else
    ifxo::DotnetSort<int, ByValue> s{by}; s.sort(idx.data(), n);
#endif
    for (int i = 0; i < n; i++) printf("%d\n", idx[i]);
    return 0;
}
