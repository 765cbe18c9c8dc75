// dm_format_host.h -- compiles a MatcherParser log_format + `<*>` templates into the device's
// DmFormat program (dm_kernels_format.cuh) and binds the configured monitors to it.  Host
// C++ only; shared by libdmdetect (dm_set_format) and the CPU emulator harness of tests/.
#pragma once
#include <cctype>
#include <cstring>
#include <string>
#include <vector>

namespace dm_format_detail {
struct FmtBuilder {
    DmFormat f;
    uint32_t n_lits = 0, pool_used = 0;
    std::vector<std::string> header_names;
    const char* err = nullptr;

    bool add_literal(const std::string& lit) {
        if (n_lits >= DM_FMT_MAX_LITS) { err = "too many literals over the log_format and the templates"; return false; }
        if (lit.size() > DM_FMT_MAX_LIT_LEN) { err = "a literal between two captures is longer than 255 bytes"; return false; }
        const uint32_t words = (uint32_t)(lit.size() + 3) / 4;
        if (pool_used + words > DM_FMT_POOL_WORDS) { err = "the literal text of log_format + templates exceeds 4096 bytes"; return false; }
        f.lit_off[n_lits] = (uint16_t)pool_used;
        f.lit_len[n_lits] = (uint8_t)lit.size();
        for (size_t i = 0; i < lit.size(); ++i)
            f.pool[pool_used + i / 4] |= (uint32_t)(uint8_t)lit[i] << (8 * (i % 4));
        pool_used += words;
        ++n_lits;
        return true;
    }

    // R-norm on one literal of a template (DESIGN.md): the bytes DmFormat.norm_drop names are
    // dropped, upper-case ASCII letters are folded when DM_NORM_LOWERCASE is set
    std::string normalised(const std::string& lit) const {
        if (!f.norm_flags) return lit;
        std::string o;
        for (unsigned char c : lit) {
            if ((f.norm_drop[c >> 5] >> (c & 31)) & 1u) continue;
            if ((f.norm_flags & DM_NORM_LOWERCASE) && c >= 'A' && c <= 'Z') c = (unsigned char)(c + 32);
            o.push_back((char)c);
        }
        return o;
    }

    // text = L0 C0 L1 C1 ...; named: captures are <Name> (name = [A-Za-z0-9_]+), else the token <*>
    // (templates, named == false, are normalised literal by literal)
    bool add_chain(const std::string& text, bool named, std::vector<std::string>* names) {
        const uint32_t c = f.n_chains;
        if (c >= DM_FMT_MAX_CHAINS) { err = "too many templates (at most 63)"; return false; }
        f.chain_first[c] = (uint16_t)n_lits;
        std::string lit;
        uint32_t lits_here = 0;
        bool last_was_capture = false;
        size_t i = 0;
        while (i < text.size()) {
            size_t cap_end = std::string::npos;
            std::string name;
            if (text[i] == '<') {
                if (!named) {
                    if (text.compare(i, 3, "<*>") == 0) cap_end = i + 3;
                } else {
                    size_t j = i + 1;
                    while (j < text.size() && (isalnum((unsigned char)text[j]) || text[j] == '_')) ++j;
                    if (j > i + 1 && j < text.size() && text[j] == '>') { cap_end = j + 1; name = text.substr(i + 1, j - i - 1); }
                }
            }
            if (cap_end == std::string::npos) { lit.push_back(text[i]); ++i; last_was_capture = false; continue; }
            if (last_was_capture) { err = "two captures with nothing between them"; return false; }
            if (!named) lit = normalised(lit);
            if (lits_here > 0 && lit.empty()) { err = "normalisation leaves nothing between two wildcards"; return false; }
            if (!add_literal(lit)) return false;                   // the literal in front of this capture (L0 may be empty)
            ++lits_here;
            lit.clear();
            if (names) names->push_back(name);
            last_was_capture = true;
            i = cap_end;
        }
        if (!named) lit = normalised(lit);
        if (last_was_capture || (!named && f.norm_flags && lits_here > 0 && lit.empty())) {
            f.chain_endcap[c] = 1;                                 // (`... <*>'` normalised: the last wildcard runs to the end)
        } else {
            if (!add_literal(lit)) return false;                   // the final literal (or the whole text)
            ++lits_here;
            f.chain_endcap[c] = 0;
        }
        const uint32_t caps_here = f.chain_endcap[c] ? lits_here : lits_here - 1;
        if (caps_here > DM_FMT_MAX_CAPTURES) { err = "more than 32 captures in one log_format / template"; return false; }
        f.n_chains = c + 1;
        f.chain_first[c + 1] = (uint16_t)n_lits;
        return true;
    }
};
}  // namespace dm_format_detail

// Returns false and sets *err on a configuration error.
inline bool dm_format_build(const char* log_format, const char* content_name, uint32_t n_templates,
                            const char* const* templates, uint32_t norm_flags, const DmMonitors& hm, DmFormat* out,
                            std::string* err) {
    dm_format_detail::FmtBuilder b;
    memset(&b.f, 0, sizeof(DmFormat));
    if (norm_flags & ~(DM_NORM_REMOVE_SPACES | DM_NORM_REMOVE_PUNCTUATION | DM_NORM_LOWERCASE)) { *err = "unknown normalisation flag"; return false; }
    b.f.norm_flags = norm_flags;
    for (unsigned c = 0; c < 128; ++c) {
        const bool space = (c >= 0x09 && c <= 0x0D) || c == 0x20;
        const bool punct = (c >= 0x21 && c <= 0x2F) || (c >= 0x3A && c <= 0x40) || (c >= 0x5B && c <= 0x60) || (c >= 0x7B && c <= 0x7E);
        if ((space && (norm_flags & DM_NORM_REMOVE_SPACES)) || (punct && (norm_flags & DM_NORM_REMOVE_PUNCTUATION)))
            b.f.norm_drop[c >> 5] |= 1u << (c & 31);
    }
    if (!b.add_chain(log_format, true, &b.header_names)) { *err = std::string("log_format: ") + b.err; return false; }
    for (size_t i = 0; i < b.header_names.size(); ++i)
        for (size_t j = 0; j < i; ++j)
            if (b.header_names[i] == b.header_names[j]) { *err = "log_format: capture <" + b.header_names[i] + "> appears twice"; return false; }
    b.f.content_capture = DM_FMT_NONE;
    const std::string cn = content_name ? content_name : "Content";
    for (size_t i = 0; i < b.header_names.size(); ++i)
        if (b.header_names[i] == cn) b.f.content_capture = (uint32_t)i;
    if (n_templates && b.f.content_capture == DM_FMT_NONE) { *err = "templates given but log_format has no <" + cn + "> capture"; return false; }
    for (uint32_t t = 0; t < n_templates; ++t) {
        if (!templates[t]) { *err = "template " + std::to_string(t) + " is NULL"; return false; }
        if (!b.add_chain(templates[t], false, nullptr)) { *err = "template " + std::to_string(t) + ": " + b.err; return false; }
    }
    b.f.n_mons = hm.n;
    for (uint32_t k = 0; k < hm.n; ++k) {
        b.f.mon_event[k] = hm.m[k].event_id;
        b.f.mon_has_event[k] = hm.m[k].has_event ? 1 : 0;
        b.f.mon_source[k] = (uint8_t)hm.m[k].source;
        b.f.mon_index[k] = DM_FMT_NONE;
        if (hm.m[k].source == 0) {
            const std::string key((const char*)hm.m[k].key, hm.m[k].key_len);
            for (size_t i = 0; i < b.header_names.size(); ++i)
                if (b.header_names[i] == key) b.f.mon_index[k] = (uint8_t)i;
        } else if (hm.m[k].var_index < DM_FMT_MAX_CAPTURES) {
            b.f.mon_index[k] = (uint8_t)hm.m[k].var_index;
        }
    }
    // captures each chain has to keep for the thread-per-record kernel
    {
        DmFormat& f = b.f;
        if (f.content_capture != DM_FMT_NONE && f.n_chains > 1) f.chain_need[0] |= 1u << f.content_capture;
        for (uint32_t k = 0; k < hm.n; ++k) {
            const uint32_t idx = f.mon_index[k];
            if (idx == DM_FMT_NONE) continue;
            if (f.mon_source[k] == 0) { f.chain_need[0] |= 1u << idx; continue; }
            for (uint32_t c = 1; c < f.n_chains; ++c)
                if (!f.mon_has_event[k] || f.mon_event[k] == (int32_t)c - 1) f.chain_need[c] |= 1u << idx;
        }
        f.max_slots = 1;
        for (uint32_t c = 0; c < f.n_chains; ++c) {
            const uint32_t n = (uint32_t)__builtin_popcount(f.chain_need[c]);
            if (n > f.max_slots) f.max_slots = n;
        }
    }
    *out = b.f;
    return true;
}
