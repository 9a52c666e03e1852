// gl_generate's prefix reuse rule (gl_engine_opts.prefix_cache; engine.cu).  Host only and self-contained, so that the CPU suite
// can compile and test it on its own (tests/hostcheck/prefix_shim.cpp).
#pragma once
#include <stdint.h>

namespace gl {

// Leading positions of `prompt` whose K / V the single-sequence pages already hold: L = the longest common prefix of the prompt
// and the ids cached[0 .. n_cached), cut so that at least min_suffix prompt tokens (and always at least one: the last prompt
// token produces the first draw) are evaluated again.  The suffix then takes the same kind of prompt pass a cold call of that
// length would take.  r = max(0, min(L, n_prompt - max(min_suffix, 1))).
inline int prefix_reuse(const int32_t* prompt, int n_prompt, const int32_t* cached, int n_cached, int min_suffix) {
    const int m = n_prompt < n_cached ? n_prompt : n_cached;
    int l = 0;
    while (l < m && prompt[l] == cached[l]) ++l;
    int r = n_prompt - (min_suffix > 1 ? min_suffix : 1);
    if (l < r) r = l;
    return r > 0 ? r : 0;
}

}  // namespace gl
