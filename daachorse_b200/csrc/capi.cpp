// Host-only half of the C ABI (construction, wire format, introspection).
// The device half lives in dev_scan.cu.
#include <cstring>
#include <new>
#include <string>

#include "host.h"

namespace dach {
namespace {
thread_local std::string g_last_error;
}
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace dach

using namespace dach;

extern "C" {

int dach_abi_version(void) { return DACH_ABI_VERSION; }
const char* dach_last_error(void) { return g_last_error.c_str(); }

int dach_bytewise_build(const uint8_t* pattern_bytes, const uint64_t* pattern_offs, const uint32_t* values,
                        uint32_t n_patterns, uint8_t match_kind, uint32_t num_free_blocks, dach_pma** out) {
    if (!out) return DACH_INVALID_ARGUMENT;
    try {
        return build_automaton(false, pattern_bytes, pattern_offs, values, n_patterns, match_kind, num_free_blocks, out);
    } catch (const std::bad_alloc&) {
        set_error("out of memory");
        return DACH_AUTOMATON_SCALE;
    }
}

int dach_charwise_build(const uint8_t* pattern_bytes, const uint64_t* pattern_offs, const uint32_t* values,
                        uint32_t n_patterns, uint8_t match_kind, uint32_t num_free_blocks, dach_pma** out) {
    if (!out) return DACH_INVALID_ARGUMENT;
    try {
        return build_automaton(true, pattern_bytes, pattern_offs, values, n_patterns, match_kind, num_free_blocks, out);
    } catch (const std::bad_alloc&) {
        set_error("out of memory");
        return DACH_AUTOMATON_SCALE;
    }
}

int dach_pma_deserialize(const uint8_t* src, size_t len, int charwise, dach_pma** out, size_t* consumed) {
    if (!out) return DACH_INVALID_ARGUMENT;
    try {
        return wire_read(src, len, charwise != 0, out, consumed);
    } catch (const std::bad_alloc&) {
        set_error("out of memory");
        return DACH_INVALID_AUTOMATON;
    }
}

size_t dach_pma_serialized_bytes(const dach_pma* pma) { return pma ? wire_size(pma) : 0; }

int dach_pma_serialize(const dach_pma* pma, uint8_t* dst, size_t cap, size_t* written) {
    if (!pma || (!dst && cap)) return DACH_INVALID_ARGUMENT;
    const size_t need = wire_size(pma);
    if (written) *written = need;
    if (cap < need) {
        set_error("serialize: destination too small");
        return DACH_INVALID_ARGUMENT;
    }
    wire_write(pma, dst);
    return DACH_OK;
}

uint8_t dach_pma_match_kind(const dach_pma* pma) { return pma ? pma->match_kind : 0; }
uint32_t dach_pma_num_states(const dach_pma* pma) { return pma ? pma->num_states : 0; }
size_t dach_pma_num_elements(const dach_pma* pma) { return pma ? pma->slots() : 0; }
int dach_pma_is_charwise(const dach_pma* pma) { return pma && pma->charwise; }

// heap_bytes (src/bytewise.rs:764-770, src/charwise.rs:813-817)
size_t dach_pma_heap_bytes(const dach_pma* pma) {
    if (!pma) return 0;
    const size_t n = pma->slots(), no = pma->outputs.size();
    if (pma->charwise) return n * 16 + pma->mapper_table.size() * 4 + no * 12;
    if (is_leftmost(pma->match_kind)) return n * 8 + n * 4 + no * 12;
    return n * 12 + pma->root_table.size() * 4 + no * 12;
}

uint32_t dach_pma_max_pattern_len(const dach_pma* pma) {
    uint32_t m = 0;
    if (pma)
        for (const OutputRec& o : pma->outputs)
            if (o.length > m) m = o.length;
    return m;
}

uint32_t dach_pma_num_outputs(const dach_pma* pma) { return pma ? (uint32_t)pma->outputs.size() : 0; }

int dach_pma_outputs(const dach_pma* pma, uint32_t* values, uint32_t* lengths, uint32_t* parents, uint32_t n) {
    if (!pma || n < pma->outputs.size()) {
        set_error("dach_pma_outputs: null automaton or n below the number of output records");
        return DACH_INVALID_ARGUMENT;
    }
    for (size_t i = 0; i < pma->outputs.size(); ++i) {
        if (values) values[i] = pma->outputs[i].value;
        if (lengths) lengths[i] = pma->outputs[i].length;
        if (parents) parents[i] = pma->outputs[i].parent;
    }
    return DACH_OK;
}

void dach_pma_free(dach_pma* pma) { delete pma; }

}  // extern "C"
