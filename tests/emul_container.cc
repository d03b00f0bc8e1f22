// tests/emul_container.cc -- TEST INFRASTRUCTURE: the model-container parser (microwakeword_b200/csrc/mww_container.cc)
// called without a device, for tests/test_container.py.
#include <stdio.h>
#include <string.h>

#include "../microwakeword_b200/csrc/mww_container.h"

using namespace mww;

// Returns parse_container's code and copies its message to msg.  On success info8 = {kind, stride, pend_cap, state_elems,
// macs_per_step, arena bytes, arena entries, tc_f16} and offsets[] = the arena offset of every entry (up to max_offsets).
extern "C" int emul_parse_container(const uint8_t *blob, size_t n, long long *info8, long long *offsets, int max_offsets, char *msg,
                                    int msg_cap) {
    ModelWeights m;
    std::string err;
    const int rc = parse_container(blob, n, &m, &err);
    snprintf(msg, (size_t)msg_cap, "%s", err.c_str());
    if (rc) return rc;
    info8[0] = (long long)m.kind; info8[1] = m.G.stride; info8[2] = m.G.pend_cap; info8[3] = m.G.state_elems;
    info8[4] = m.G.macs_per_step; info8[5] = (long long)m.arena.size(); info8[6] = (long long)m.fixups.size(); info8[7] = m.tc_f16;
    for (size_t i = 0; i < m.fixups.size() && (int)i < max_offsets; ++i) {
        uintptr_t off;
        memcpy(&off, reinterpret_cast<const unsigned char *>(&m) + m.fixups[i], sizeof off);
        offsets[i] = (long long)off;
    }
    return 0;
}
