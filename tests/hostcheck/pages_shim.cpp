// TEST INFRASTRUCTURE: the KV page pool and prefix index (gridllm_b200/csrc/prefix_pages.h) compiled for the host, so that
// tests/test_prefix_pages_cpu.py can check them against a Python restatement.  Never linked into libgridllm_native.so.
#include "../../gridllm_b200/csrc/prefix_pages.h"

extern "C" {

void* pp_new(int n_pages) {
    gl::PagePool* p = new gl::PagePool();
    p->init(n_pages);
    return p;
}
void pp_delete(void* h) { delete static_cast<gl::PagePool*>(h); }

// n pages into out; returns n, or -1 when the pool cannot supply them (nothing taken)
int pp_alloc(void* h, int n, int32_t* out) {
    std::vector<int> v;
    if (!static_cast<gl::PagePool*>(h)->alloc(n, v)) return -1;
    for (int i = 0; i < n; ++i) out[i] = v[i];
    return n;
}
void pp_ref(void* h, int page) { static_cast<gl::PagePool*>(h)->ref(page); }
void pp_release(void* h, int page) { static_cast<gl::PagePool*>(h)->release(page); }
int pp_match(void* h, const int32_t* ids, int n, int32_t* out) {
    std::vector<int> v;
    const int l = static_cast<gl::PagePool*>(h)->match(ids, n, &v);
    for (int i = 0; i < l; ++i) out[i] = v[i];
    return l;
}
int pp_insert(void* h, int parent, const int32_t* ids16, int page) { return static_cast<gl::PagePool*>(h)->insert(parent, ids16, page) ? 1 : 0; }
void pp_forget(void* h, int page) { static_cast<gl::PagePool*>(h)->forget(page); }
// out[0] free pages, out[1] retained pages; then per page refs and indexed
void pp_state(void* h, int32_t* counts, int32_t* refs, int32_t* indexed) {
    const gl::PagePool* p = static_cast<gl::PagePool*>(h);
    counts[0] = p->free_count();
    counts[1] = p->retained_count();
    for (int i = 0; i < p->pool(); ++i) {
        refs[i] = p->refs(i);
        indexed[i] = p->indexed(i) ? 1 : 0;
    }
}
int pp_reuse(int matched_pages, int n_prompt, int prefill_min) { return gl::shared_prefix_reuse(matched_pages, n_prompt, prefill_min); }

}
