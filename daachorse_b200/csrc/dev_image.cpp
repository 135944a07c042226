// Builds the device scan image from a validated host automaton.
//
// Results of a scan depend only on the automaton's transition/output structure, never on
// where the builder placed a state (SURVEY.md Appendix C.3), so the image is free to carry
// derived fields next to the reference's BASE / CHECK / FAIL / OUTPUT_POS values.
#include "dev_image.h"

#include <algorithm>

namespace dach {

namespace {

// Every failure chain must end at ROOT (or at DEAD where DEAD is a terminal).  O(n).
bool fail_chains_terminate(const dach_pma* p, bool dead_is_terminal) {
    const size_t n = p->slots();
    std::vector<uint8_t> color(n, 0);  // 0 new, 1 on the current path, 2 proven
    std::vector<uint32_t> path;
    for (size_t start = 0; start < n; ++start) {
        if (color[start]) continue;
        path.clear();
        uint32_t s = uint32_t(start);
        for (;;) {
            if (s == kRoot || (dead_is_terminal && s == kDead) || color[s] == 2) break;
            if (color[s] == 1) return false;  // cycle
            color[s] = 1;
            path.push_back(s);
            s = p->fail[s];
        }
        for (uint32_t v : path) color[v] = 2;
    }
    return true;
}


// ---- hot-first relayout of the bytewise double array (compact image only) --------------------------
//
// Scan results do not depend on where a state sits (SURVEY.md Appendix C.3), only the wire format has to
// keep the crate's numbering.  The compact image therefore moves the children of the states the text
// visits most into a dense *hot region* at the front of the array, placed hottest first, so that
//   * the leading records can be staged in shared memory and served without a tag ("slot < hot_n"),
//   * what does not fit there still shares L1 lines and L2 sectors with other hot records.
// Hotness is a property of the automaton alone: failure transitions keep a scan near the top of the trie,
// so parents are ranked by depth, then by subtree size per child (on the C3 bench text this static order
// covers 60.8 % of all landings with 8192 slots; ranking by measured visit counts covers 61.4 %).
// Children of one parent stay an XOR family (slot = BASE ^ label), they are re-placed first-fit with a
// new BASE inside the region; everything else keeps its slot, shifted up by the region size H (a multiple
// of 256, so (BASE + H) ^ c == (BASE ^ c) + H).  ROOT and DEAD keep ids 0 and 1.
struct Relayout {
    uint32_t hot_slots = 0;             // H; 0 = identity
    std::vector<uint32_t> new_of_old;   // slot in the crate's numbering -> slot in the compact image
    std::vector<uint32_t> new_base;     // BASE of every (old) slot in the compact image's numbering
    std::vector<uint32_t> sig;          // child signature per (old) slot
    std::vector<uint32_t> vacant_check; // per region slot: 0x100 | CHECK for slots no state occupies (and ROOT, DEAD)
    bool textbook = false;              // Standard automata: the trie and its failure links are Aho-Corasick's (see below)
    uint32_t max_depth = 0;             // depth of the deepest trie state
};

constexpr uint32_t kNone = 0xffffffffu;

void relayout_bytewise(const dach_pma* p, uint32_t want_hot_slots, Relayout* R) {
    const size_t n = p->slots();
    R->hot_slots = 0;
    R->textbook = false;
    R->max_depth = 0;
    R->new_of_old.resize(n);
    R->new_base.assign(p->base.begin(), p->base.end());
    R->sig.assign(n, 0);
    for (size_t s = 0; s < n; ++s) R->new_of_old[s] = uint32_t(s);
    if (n < 2) return;

    // trie walk from ROOT: parent, depth, number of children, BFS order, child signatures
    std::vector<uint32_t> parent(n, kNone), depth(n, 0), nchild(n, 0), bfs;
    bfs.reserve(n);
    bfs.push_back(kRoot);
    parent[kRoot] = kRoot;
    bool tree = true;  // every slot is the child of at most one state (always true for automata the builders make)
    for (size_t h = 0; h < bfs.size(); ++h) {
        const uint32_t s = bfs[h];
        const uint32_t b = p->base[s];
        if (b == 0) continue;
        uint32_t sig = 0, k = 0;
        for (uint32_t c = 0; c < 256; ++c) {
            const uint32_t ci = b ^ c;
            if (ci >= n || (p->opos_ch[ci] & 0xffu) != c) continue;
            sig |= 1u << (c & 31);
            if (ci == kRoot || ci == kDead || parent[ci] != kNone) {
                tree = false;
                continue;
            }
            parent[ci] = s;
            depth[ci] = depth[s] + 1;
            bfs.push_back(ci);
            ++k;
        }
        R->sig[s] = sig;
        nchild[s] = k;
    }
    // Slots the walk did not reach still get their signature.  In an automaton the builders made these are
    // vacant and have no BASE.  A hand-made one may hold states there that only failure links lead to; if such
    // a state answers to children, they are some trie state's children as well (or garbage), and moving that
    // family away would change what the failure walk finds: the layout is then left alone.
    for (size_t s = 0; s < n; ++s) {
        if (parent[s] != kNone || p->base[s] == 0) continue;
        uint32_t sig = 0;
        for (uint32_t c = 0; c < 256; ++c) {
            const uint32_t ci = p->base[s] ^ c;
            if (ci < n && (p->opos_ch[ci] & 0xffu) == c) sig |= 1u << (c & 31);
        }
        R->sig[s] = sig;
        if (sig) tree = false;
    }
    // Is this the automaton Aho and Corasick describe -- every state with children a trie state, every failure
    // link the state of the longest proper suffix?  Always, for what the builders make (src/nfa_builder.rs).  A
    // hand-made blob can pass the crate's validation without it; then the state after a text is no longer a
    // function of the text's last bytes, which cutting long haystacks into segments relies on (dev_scan.cu).
    if (tree && !is_leftmost(p->match_kind)) {
        bool ok = true;
        for (size_t h = 1; h < bfs.size() && ok; ++h) {
            const uint32_t s = bfs[h], par = parent[s], c = p->opos_ch[s] & 0xffu;
            if (depth[s] > R->max_depth) R->max_depth = depth[s];
            uint32_t t = kRoot;
            if (par != kRoot) {
                t = p->fail[par];
                for (;;) {  // the crate's transition from the parent's failure state (src/bytewise.rs:1063-1088)
                    const uint32_t b = p->base[t], ci = b ^ c;
                    if (b != 0 && ci < n && (p->opos_ch[ci] & 0xffu) == c) {
                        t = ci;
                        break;
                    }
                    if (t == kRoot) break;
                    t = p->fail[t];
                }
            }
            ok = p->fail[s] == t;
        }
        R->textbook = ok;
    }
    uint64_t H64 = std::min<uint64_t>(want_hot_slots, (uint64_t(n) + 255) & ~uint64_t(255));
    H64 &= ~uint64_t(255);
    if (!tree || H64 == 0 || n + H64 > (size_t(1) << 24)) return;
    const uint32_t H = uint32_t(H64);

    // subtree sizes (states below and including s), children before parents
    std::vector<uint32_t> sub(n, 0);
    for (size_t h = bfs.size(); h-- > 0;) {
        const uint32_t s = bfs[h];
        sub[s] += 1;
        if (s != kRoot) sub[parent[s]] += sub[s];
    }
    // parents, hottest first: by depth, then by subtree size per child
    std::vector<uint32_t> par;
    for (uint32_t s : bfs)
        if (nchild[s]) par.push_back(s);
    std::stable_sort(par.begin(), par.end(), [&](uint32_t a, uint32_t b) {
        if (depth[a] != depth[b]) return depth[a] < depth[b];
        return uint64_t(sub[a]) * nchild[b] > uint64_t(sub[b]) * nchild[a];
    });

    // first-fit placement inside [0, H): slots 0 and 1 stay ROOT and DEAD; BASE values are unique and non-zero
    std::vector<uint8_t> used(H, 0), base_used(H, 0);
    used[kRoot] = used[kDead] = 1;
    base_used[0] = 1;
    uint32_t first_free = 2, n_free = H - 2, fails = 0;
    std::vector<uint8_t> labels, moved(n, 0);  // moved: the slot (a child) / the BASE (a parent) was re-placed
    std::vector<uint8_t> rebased(n, 0);
    for (uint32_t s : par) {
        if (n_free == 0 || fails >= 256) break;
        if (nchild[s] > n_free) {
            ++fails;
            continue;
        }
        labels.clear();
        const uint32_t b_old = p->base[s];
        for (uint32_t c = 0; c < 256; ++c) {
            const uint32_t ci = b_old ^ c;
            if (ci < n && parent[ci] == s && (p->opos_ch[ci] & 0xffu) == c) labels.push_back(uint8_t(c));
        }
        while (first_free < H && used[first_free]) ++first_free;
        uint32_t found = kNone;
        for (uint32_t v = first_free; v < H; ++v) {
            if (used[v]) continue;
            const uint32_t b = v ^ labels[0];
            if (base_used[b]) continue;
            bool ok = true;
            for (uint8_t c : labels)
                if (used[b ^ c]) {
                    ok = false;
                    break;
                }
            if (ok) {
                found = b;
                break;
            }
        }
        if (found == kNone) {
            ++fails;
            continue;
        }
        fails = 0;
        base_used[found] = 1;
        R->new_base[s] = found;
        rebased[s] = 1;
        for (uint8_t c : labels) {
            used[found ^ c] = 1;
            R->new_of_old[b_old ^ c] = found ^ c;
            moved[b_old ^ c] = 1;
            --n_free;
        }
    }
    // everything else: old slot + H (ROOT and DEAD keep 0 and 1), BASE + H
    for (size_t s = 0; s < n; ++s) {
        if (s != kRoot && s != kDead && !moved[s]) R->new_of_old[s] = uint32_t(s) + H;
        if (!rebased[s] && p->base[s] != 0) R->new_base[s] = p->base[s] + H;
    }
    // Vacant slots of the region (and ROOT / DEAD, which no probe may ever hit) get the CHECK of a BASE that
    // no state of their 256-block uses, like src/bytewise/builder.rs:389-399 does for closed blocks.
    R->vacant_check.assign(H, 0);
    for (uint32_t blk = 0; blk < H; blk += 256) {
        uint32_t ub = blk == 0 ? 0u : kNone;  // BASE 0 means "no children": never a real BASE
        for (uint32_t b = blk; ub == kNone && b < blk + 256; ++b)
            if (!base_used[b]) {
                ub = b;
                break;
            }
        for (uint32_t v = blk; v < blk + 256; ++v)
            if (!used[v] || v == kRoot || v == kDead) R->vacant_check[v] = ub == kNone ? 0x100u : (0x100u | ((ub ^ v) & 0xffu));
    }
    R->hot_slots = H;
}

}  // namespace

int build_image(const dach_pma* p, HostImage* img) {
    const size_t n = p->slots();
    const bool lm = is_leftmost(p->match_kind);
    img->charwise = p->charwise;
    img->match_kind = p->match_kind;
    img->n_slots = uint32_t(n);
    img->root_opos = n ? p->state_output_pos(kRoot) : 0;
    img->max_pattern_len = 0;
    for (const OutputRec& o : p->outputs)
        if (o.length > img->max_pattern_len) img->max_pattern_len = o.length;

    if (n >= 0x80000000ull) {
        set_error("automaton too large for the device image (2^31 slots)");
        return DACH_AUTOMATON_SCALE;
    }
    if (!fail_chains_terminate(p, p->charwise || lm)) {
        set_error("invalid automaton: a failure chain never reaches the root");
        return DACH_INVALID_AUTOMATON;
    }

    img->outputs.resize(p->outputs.size() * 4);
    for (size_t i = 0; i < p->outputs.size(); ++i) {
        img->outputs[i * 4 + 0] = p->outputs[i].value;
        img->outputs[i * 4 + 1] = p->outputs[i].length;
        img->outputs[i * 4 + 2] = p->outputs[i].parent;
        // the length of the list that starts here (this record and its parents): what a count of
        // find_overlapping adds per event without walking the list.  A parent comes before its child
        // (deserialize checks parent < own 1-based index), so it is known already.
        const uint32_t par = p->outputs[i].parent;
        img->outputs[i * 4 + 3] = 1u + (par ? img->outputs[(size_t)(par - 1) * 4 + 3] : 0u);
    }
    // two-entry lists (k_expand_desc): the record and its parent in one 16-byte entry, the list length's class in
    // the top two bits of the parent's length.  Only if no pattern length reaches those bits.
    img->pairs.clear();
    if (img->max_pattern_len < PAIR_LEN_MASK) {
        img->pairs.resize(p->outputs.size() * 4);
        for (size_t i = 0; i < p->outputs.size(); ++i) {
            const uint32_t par = p->outputs[i].parent, len = img->outputs[i * 4 + 3];
            img->pairs[i * 4 + 0] = p->outputs[i].value;
            img->pairs[i * 4 + 1] = p->outputs[i].length;
            img->pairs[i * 4 + 2] = par ? p->outputs[par - 1].value : 0u;
            img->pairs[i * 4 + 3] = (par ? p->outputs[par - 1].length : 0u) | (len < 3u ? len : 3u) << PAIR_CLASS_SHIFT;
        }
    }

    img->rec.resize(n * 4);
    if (!p->charwise) {
        auto skip_leaves = [&](uint32_t f) {  // failure target with child-less states skipped
            while (f != kRoot && !(lm && f == kDead) && p->base[f] == 0) f = p->fail[f];
            return f;
        };
        for (size_t s = 0; s < n; ++s) {
            const uint32_t f = skip_leaves(p->fail[s]);
            const bool terminal = f == kRoot || (lm && f == kDead);
            uint32_t* r = &img->rec[s * 4];
            r[0] = p->base[s];
            r[1] = f;
            r[2] = terminal ? 0 : p->base[f];
            // bit 31: the failure state's own (leaf-skipped) failure target is ROOT
            if (!terminal && !lm && skip_leaves(p->fail[f]) == kRoot) r[2] |= 0x80000000u;
            r[3] = p->opos_ch[s];
        }
        // dense ROOT row; also valid for the leftmost automaton, whose ROOT transition is
        // "child or stay" (src/bytewise.rs:1102-1117)
        img->root_table.assign(256, kRoot);
        if (n && p->base[kRoot] != 0) {
            const uint32_t b = p->base[kRoot];
            for (uint32_t c = 0; c < 256; ++c) {
                const uint32_t ci = b ^ c;
                if (ci < n && (p->opos_ch[ci] & 0xff) == c) img->root_table[c] = ci;
            }
        }
        // compact image for the lane-machine kernels (automata of at most 2^24 slots), hot-first relayout
        img->root_base = n ? p->base[kRoot] : 0;
        img->hot_slots = 0;
        if (n <= (size_t(1) << 24) && p->outputs.size() < (size_t(1) << 24)) {
            Relayout R;
            relayout_bytewise(p, img->want_hot_slots, &R);
            img->segmentable = R.textbook && R.max_depth <= img->max_pattern_len;
            const uint32_t H = R.hot_slots;
            const size_t N = n + H;
            img->hot_slots = H;
            img->n_cslots = uint32_t(N);
            img->crec.assign(N * 4, 0);
            img->opos_tab.assign(N, 0);
            img->new_of_old = R.new_of_old;
            img->old_of_new.assign(N, kRoot);
            img->root_base = n ? R.new_base[kRoot] : 0;
            auto nid = [&](uint32_t s) { return s < n ? R.new_of_old[s] : s; };
            for (size_t s = 0; s < n; ++s) {
                const uint32_t* w = &img->rec[s * 4];
                const uint32_t ns = R.new_of_old[s];
                img->old_of_new[ns] = uint32_t(s);
                uint32_t* r = &img->crec[size_t(ns) * 4];
                const uint32_t opos = p->opos_ch[s] >> 8;
                const uint32_t f = w[1];  // leaf-skipped failure target (crate numbering)
                const bool terminal = f == kRoot || (lm && f == kDead);
                uint32_t flags = opos ? 1u : 0u;
                uint32_t fbase = terminal ? 0u : R.new_base[f];
                if (!lm) {
                    if (w[2] & 0x80000000u) flags |= 2u;  // CF_F2ROOT
                    if (f == kRoot) flags |= 8u, fbase = img->root_base;  // CF_FROOT: fbase pre-resolved to BASE(ROOT)
                } else if (!terminal) {
                    const uint32_t f2 = skip_leaves(p->fail[f]);
                    if (f2 == kRoot) flags |= 2u;  // CF_F2ROOT
                    if (f2 == kDead) flags |= 4u;  // CF_F2DEAD
                }
                uint32_t check = p->opos_ch[s] & 0xffu;
                if (ns < H && R.vacant_check[ns]) check = R.vacant_check[ns] & 0xffu;  // ROOT, DEAD
                r[0] = (R.new_base[s] << 8) | check;
                r[1] = (nid(f) << 8) | flags;
                // low byte: the length of the state's output list, saturated at 255 (StdMachine3 queues it with
                // the event, so that its drain needs neither output_pos nor the list)
                const uint32_t list = opos ? img->outputs[(size_t)(opos - 1) * 4 + 3] : 0u;
                r[2] = (fbase << 8) | std::min<uint32_t>(list, 255u);
                r[3] = R.sig[s];
                img->opos_tab[ns] = opos;
            }
            for (uint32_t v = 0; v < H; ++v)  // slots of the region no state occupies
                if (R.vacant_check[v] && v != kRoot && v != kDead) img->crec[size_t(v) * 4] = R.vacant_check[v] & 0xffu;
            // Slots a moved state left behind (ROOT's and DEAD's old places included) keep its CHECK byte: the
            // shifted part is then probe for probe the crate's array, and the only BASE a moved child's byte
            // could answer to is its parent's old one, which moved with the family and is unique.  (An all-zero
            // record would answer label 0 to whichever state's BASE equals the slot: a wrong transition on a
            // NUL byte.)
            if (H)
                for (size_t s = 0; s < n; ++s)
                    if (R.new_of_old[s] < H) img->crec[(s + H) * 4] = p->opos_ch[s] & 0xffu;
        }
    } else {
        for (size_t s = 0; s < n; ++s) {
            uint32_t* r = &img->rec[s * 4];
            r[0] = p->base[s];
            r[1] = p->check[s];
            r[2] = p->fail[s];
            r[3] = p->output_pos[s];
        }
        img->root_table.assign(256, kRoot);  // unused by the charwise kernels
        img->mapper = p->mapper_table;
        // compact image for the charwise lane machine (scan_lane.cuh, CwMachine)
        img->root_base = n ? p->base[kRoot] : 0;
        if (n < (size_t(1) << 24) && p->outputs.size() < (size_t(1) << 24)) {
            auto skip_leaves = [&](uint32_t f) {  // failure target with child-less states skipped
                while (f != kRoot && f != kDead && p->base[f] == 0) f = p->fail[f];
                return f;
            };
            // child signatures: bit (mapped code & 15) of the parent for every occupied slot
            std::vector<uint32_t> sig(n, 0);
            for (size_t s = 0; s < n; ++s) {
                const uint32_t par = p->check[s];
                if (par >= n || p->base[par] == 0) continue;
                const uint32_t code = uint32_t(s) ^ p->base[par];
                if (code < p->alphabet_size) sig[par] |= 1u << (code & 15);
            }
            img->crec.resize(n * 4);
            img->opos_tab.resize(n);
            for (size_t s = 0; s < n; ++s) {
                const uint32_t f = skip_leaves(p->fail[s]);
                const bool terminal = f == kRoot || f == kDead;
                uint32_t flags = p->output_pos[s] ? 1u : 0u;
                if (!terminal) {
                    const uint32_t f2 = skip_leaves(p->fail[f]);
                    if (f2 == kRoot) flags |= 2u;  // CF_F2ROOT
                    if (f2 == kDead) flags |= 4u;  // CF_F2DEAD
                }
                const uint32_t chk = p->check[s] < n ? p->check[s] : 0xffffffu;  // vacant: matches no state id
                uint32_t* r = &img->crec[s * 4];
                r[0] = (p->base[s] << 8) | (sig[s] & 0xffu);
                r[1] = (f << 8) | flags;
                r[2] = ((terminal ? 0u : p->base[f]) << 8) | (sig[s] >> 8);
                r[3] = chk << 8;
                img->opos_tab[s] = p->output_pos[s];
            }
        }
    }
    return DACH_OK;
}

}  // namespace dach
