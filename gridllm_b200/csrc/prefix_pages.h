// The KV page pool (engine.cu, engine_batch.cu): reference-counted physical pages and the index of prompt-prefix pages that
// batch slots share (gl_engine_opts batch_prefix_cache).  Host only and self-contained, so that the CPU suite can compile and
// test it on its own (tests/hostcheck/pages_shim.cpp).
//
// Every page the engine hands out comes from PagePool::alloc and goes back through PagePool::release.  A page is in exactly
// one of three states:
//   free        on the free list (handed out from its back: pages come out in reverse order, so a page table is a real
//               indirection);
//   referenced  refs > 0: some sequence's table holds it;
//   retained    refs == 0 but indexed: it still holds the K / V of a prompt prefix a later sequence may share.
// alloc takes free pages first, then evicts retained pages: the least recently released LEAF first (a page no other indexed
// page chains from).  It fails only when free + retained pages are too few, i.e. when live references hold the pool.
//
// The index is a trie of FULL pages: node = (parent page or -1, the 16 token ids of the page) -> the page whose K / V rows are
// those 16 positions after exactly that id prefix.  Ids are compared exactly; the hash only finds candidates.  A sequence
// indexes its pages in order, each under its own previous page, and stops at the first key the index already has, so an
// indexed page's parent is referenced by every sequence that references the page: a retained page's whole subtree is retained,
// and free + retained pages are really available.
#pragma once
#include <stdint.h>

#include <set>
#include <unordered_map>
#include <utility>
#include <vector>

namespace gl {

constexpr int PP_PAGE_TOKENS = 16;      // = KV_PAGE_TOKENS

// Positions of a prompt taken from shared pages when the index holds a chain of `matched_pages` pages that matches it: whole
// pages, and at least max(prefill_min, 1) prompt tokens are evaluated, so the suffix takes the same kind of prompt pass a cold
// open of that length takes.  r = 16 floor(min(16 L, n_prompt - max(prefill_min, 1)) / 16), never negative.
inline int shared_prefix_reuse(int matched_pages, int n_prompt, int prefill_min) {
    int r = n_prompt - (prefill_min > 1 ? prefill_min : 1);
    if (PP_PAGE_TOKENS * matched_pages < r) r = PP_PAGE_TOKENS * matched_pages;
    return r > 0 ? r / PP_PAGE_TOKENS * PP_PAGE_TOKENS : 0;
}

class PagePool {
public:
    void init(int n_pages) {
        node_.assign(n_pages, Node{});
        free_.resize(n_pages);
        for (int i = 0; i < n_pages; ++i) free_[i] = i;
        leaves_.clear();
        index_.clear();
        retained_ = 0;
        clock_ = 0;
    }
    int pool() const { return (int)node_.size(); }
    int free_count() const { return (int)free_.size(); }
    int retained_count() const { return retained_; }
    int available() const { return (int)free_.size() + retained_; }        // what alloc can hand out
    int refs(int p) const { return node_[p].refs; }
    bool indexed(int p) const { return node_[p].indexed; }

    // n pages with one reference each, appended to out; false (nothing taken) when fewer than n are free or retained
    bool alloc(int n, std::vector<int>& out) {
        if (n > available()) return false;
        for (int i = 0; i < n; ++i) {
            int p;
            if (!free_.empty()) {
                p = free_.back();
                free_.pop_back();
            } else {
                p = leaves_.begin()->second;                                 // least recently released retained leaf
                leaves_.erase(leaves_.begin());
                --retained_;
                unindex(p);
            }
            node_[p].refs = 1;
            out.push_back(p);
        }
        return true;
    }
    // one more reference to an indexed page (a sequence that shares it); a retained page stops being evictable
    void ref(int p) {
        Node& n = node_[p];
        if (n.refs == 0 && n.indexed) {
            --retained_;
            if (n.children == 0) leaves_.erase({n.stamp, p});
        }
        ++n.refs;
    }
    // drop one reference: at zero an indexed page is retained (most recently released), any other page is free again
    void release(int p) {
        Node& n = node_[p];
        if (--n.refs > 0) return;
        if (n.indexed) {
            ++retained_;
            n.stamp = ++clock_;
            if (n.children == 0) leaves_.insert({n.stamp, p});
        } else {
            free_.push_back(p);
        }
    }

    // the longest chain of indexed pages matching ids[0 .. n_ids): its pages go to *pages (when not null), the count is returned
    int match(const int32_t* ids, int n_ids, std::vector<int>* pages) const {
        int parent = -1, l = 0;
        for (; (l + 1) * PP_PAGE_TOKENS <= n_ids; ++l) {
            const int p = find(parent, ids + l * PP_PAGE_TOKENS);
            if (p < 0) break;
            if (pages) pages->push_back(p);
            parent = p;
        }
        return l;
    }
    // index `page` (referenced, not yet indexed) as the page after `parent` (-1: the first page) holding ids16; false, and
    // nothing changes, when that key is already indexed
    bool insert(int parent, const int32_t* ids16, int page) {
        if (find(parent, ids16) >= 0) return false;
        Node& n = node_[page];
        n.indexed = true;
        n.parent = parent;
        n.children = 0;
        for (int i = 0; i < PP_PAGE_TOKENS; ++i) n.ids[i] = ids16[i];
        index_.insert({key(parent, ids16), page});
        if (parent >= 0) ++node_[parent].children;
        return true;
    }
    // take a referenced leaf back out of the index (a pass that failed after its pages were indexed)
    void forget(int page) {
        if (node_[page].indexed && node_[page].children == 0) unindex(page);
    }

private:
    struct Node {
        int refs = 0;
        bool indexed = false;
        int parent = -1;
        int children = 0;            // indexed pages whose parent this is
        uint64_t stamp = 0;          // release clock (retained pages)
        int32_t ids[PP_PAGE_TOKENS] = {};
    };
    static uint64_t key(int parent, const int32_t* ids16) {
        uint64_t h = 0x9e3779b97f4a7c15ull ^ (uint64_t)(uint32_t)parent;
        for (int i = 0; i < PP_PAGE_TOKENS; ++i) {
            h ^= (uint64_t)(uint32_t)ids16[i];
            h *= 0x100000001b3ull;
            h ^= h >> 29;
        }
        return h;
    }
    int find(int parent, const int32_t* ids16) const {
        auto range = index_.equal_range(key(parent, ids16));
        for (auto it = range.first; it != range.second; ++it) {
            const Node& n = node_[it->second];
            if (n.parent != parent) continue;
            bool same = true;
            for (int i = 0; i < PP_PAGE_TOKENS && same; ++i) same = n.ids[i] == ids16[i];
            if (same) return it->second;
        }
        return -1;
    }
    // out of the index; a retained parent left without children becomes an evictable leaf
    void unindex(int p) {
        Node& n = node_[p];
        auto range = index_.equal_range(key(n.parent, n.ids));
        for (auto it = range.first; it != range.second; ++it)
            if (it->second == p) { index_.erase(it); break; }
        if (n.parent >= 0) {
            Node& par = node_[n.parent];
            if (--par.children == 0 && par.refs == 0 && par.indexed) leaves_.insert({par.stamp, n.parent});
        }
        n.indexed = false;
        n.parent = -1;
        n.children = 0;
    }

    std::vector<Node> node_;                          // per physical page
    std::vector<int> free_;
    std::set<std::pair<uint64_t, int>> leaves_;       // retained leaves by release stamp (oldest first)
    std::unordered_multimap<uint64_t, int> index_;    // key hash -> indexed pages
    int retained_ = 0;
    uint64_t clock_ = 0;
};

}  // namespace gl
