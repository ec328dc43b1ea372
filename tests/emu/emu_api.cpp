// TEST-ONLY host emulation of the infidex_b200 kernels (Ctx == one host thread). The product's host driver runs unchanged and
// its launch shim calls the kernels as host functions, so the CPU test suite checks the launch sequence and the kernel logic,
// from the device-side index build to the final results, against the oracle without a GPU. Never loaded by the product package.
#define IFX_EMU 1
#include "../../infidex_b200/csrc/ifx_api.inl"

// ---- test hooks (tests/test_cov_shortcuts.py): the exact shortcuts of the coverage kernel next to the row-based Damerau they replace ----
extern "C" int ifx_emu_damerau(const uint16_t* s, int ns, const uint16_t* t, int nt, int maxd) {      // all units < 128: the character tables are not consulted
    static ifx::DevIndex ix{}; return ifx::damerau(ix, ifx::Str{s, ns}, ifx::Str{t, nt}, maxd, true);
}
extern "C" int ifx_emu_damerau1_ascii(const uint16_t* s, int ns, const uint16_t* t, int nt) { return ifx::damerau1_ascii(ifx::Str{s, ns}, ifx::Str{t, nt}); }
extern "C" int ifx_emu_sig_far(const uint16_t* s, int ns, const uint16_t* t, int nt, int k) {
    static ifx::DevIndex ix{}; return ifx::sig_far(ifx::fold_sig(ix, ifx::Str{s, ns}), ifx::fold_sig(ix, ifx::Str{t, nt}), k) ? 1 : 0;
}
