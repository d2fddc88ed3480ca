// Shape gate shared by the persistent conv entry points (bm_tc_conv1d_persistent, bm_tc_conv1d_f16): the column-half
// rule nh in {160, 128} of the library's published contract.
#pragma once
#include "tc_common.cuh"

namespace bm {
namespace tc {

inline int pair_pick_nh(int Ntot, int glu) {
    if (glu && (Ntot % 2)) return 0;
    const int n = glu ? Ntot / 2 : Ntot;
    for (int nh = 160; nh >= 128; nh -= 32) {
        const int per_tile = glu ? nh : 2 * nh;
        if (n % per_tile == 0) return nh;
    }
    return 0;
}
inline bool pair_conv_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    if (Kw < 1 || Kw > 3 || (Kw & 1) == 0) return false;
    if (Cin % 32 != 0) return false;
    return pair_pick_nh(Ntot, glu) != 0;
}

}  // namespace tc
}  // namespace bm
