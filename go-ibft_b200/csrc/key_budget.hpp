// key_budget.hpp -- the key registry's comb-table budget (ibft_set_key_table_budget): which registry entries hold one of the
// max_tables comb-table slots, and which slot.  Host-only C++ (no CUDA), so that the policy can be tested on the CPU.
//
// A budget decides only at RECLAIM POINTS (every lane held, device drained): the entries with a known key that a resident table
// lists are ranked by
//   1. the reclaim point at which the known-key pass last looked them up (newest first),
//   2. entries that hold a table now before those that do not (when everybody is equally hot, nothing churns),
//   3. address, ascending,
// and the first max_tables keep or get a table.  Between reclaim points, table slots left free may be given to keys learned
// since (take_free); nothing is ever taken away from an entry there.
#pragma once

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <set>
#include <vector>

namespace ibft {

constexpr uint32_t kNoTable = 0xFFFFFFFFu;

struct key_budget {
  uint32_t max_tables = 0;          // table slots [0, max_tables)
  uint64_t clock = 0;               // reclaim points so far
  std::vector<uint64_t> stamp;      // per entry: reclaim point at which its key was last used (0: never)
  std::vector<uint32_t> table;      // per entry: its table slot, or kNoTable
  std::vector<uint32_t> owner;      // per table slot: its entry, or kNoTable (size: the larger of the old and new budget
                                    // while a reclaim point moves tables down, max_tables otherwise)
  std::set<uint32_t> free_slots;    // slots below max_tables without an owner

  struct move { uint32_t entry, from, to; };
  struct plan {
    std::vector<uint32_t> evicted;   // entries that lost their table (known key, no table from now on)
    std::vector<uint32_t> admitted;  // entries that got a table slot (to be built)
    std::vector<uint32_t> retired;   // entries no resident table lists whose slot was freed
    std::vector<move> moves;         // kept tables that sat at or above max_tables, in copy order
  };

  void ensure(uint32_t n_entries) {
    if (table.size() < n_entries) { table.resize(n_entries, kNoTable); stamp.resize(n_entries, 0); }
  }
  uint32_t live() const { return (uint32_t)std::count_if(owner.begin(), owner.end(), [](uint32_t o) { return o != kNoTable; }); }

  // give entry r the lowest free slot; kNoTable when none is left
  uint32_t take_free(uint32_t r) {
    if (free_slots.empty()) return kNoTable;
    const uint32_t t = *free_slots.begin();
    free_slots.erase(free_slots.begin());
    owner[t] = r;
    table[r] = t;
    return t;
  }
  // entry r gives its slot back (its table could not be placed, or it left every resident table)
  void drop(uint32_t r) {
    const uint32_t t = table[r];
    if (t == kNoTable) return;
    table[r] = kNoTable;
    owner[t] = kNoTable;
    if (t < max_tables) free_slots.insert(t);
  }
  // adopt slots [0, n) as they are, slot t holding entry t when holds[t] (the pool of an engine that had no budget so far:
  // entry r's table sits in slot r)
  void adopt_identity(uint32_t n_entries, const std::vector<uint8_t>& holds) {
    ensure(n_entries);
    max_tables = (uint32_t)holds.size();
    owner.assign(holds.size(), kNoTable);
    free_slots.clear();
    for (uint32_t t = 0; t < holds.size(); t++) {
      if (holds[t] && t < n_entries) { owner[t] = t; table[t] = t; }
      else free_slots.insert(t);
    }
  }

  // One reclaim point over entries [0, n).  listed[r]: a resident table lists entry r; known[r]: its key is known; used[r]: the
  // known-key pass looked it up since the last reclaim point (the caller clears the flags); addr: 20 bytes per entry.
  plan reclaim(uint32_t n, const uint8_t* listed, const uint8_t* known, const uint8_t* used, const uint8_t* addr, uint32_t new_max) {
    plan p;
    ensure(n);
    clock++;
    for (uint32_t r = 0; r < n; r++) if (used[r]) stamp[r] = clock;
    // an entry no resident table lists is retired: it gives its slot back and forgets when it was used
    std::vector<uint32_t> cand;
    for (uint32_t r = 0; r < n; r++) {
      if (!listed[r]) {
        if (table[r] != kNoTable) { drop(r); p.retired.push_back(r); }
        stamp[r] = 0;
      } else if (known[r]) {
        cand.push_back(r);
      }
    }
    std::sort(cand.begin(), cand.end(), [&](uint32_t a, uint32_t b) {
      if (stamp[a] != stamp[b]) return stamp[a] > stamp[b];
      const bool ta = table[a] != kNoTable, tb = table[b] != kNoTable;
      if (ta != tb) return ta;
      const int c = memcmp(addr + 20 * (size_t)a, addr + 20 * (size_t)b, 20);
      return c != 0 ? c < 0 : a < b;
    });
    const size_t keep = std::min<size_t>(cand.size(), new_max);
    // entries below the cut that hold a table lose it (so do tables of entries whose key is no longer known)
    for (size_t i = keep; i < cand.size(); i++)
      if (table[cand[i]] != kNoTable) { drop(cand[i]); p.evicted.push_back(cand[i]); }
    for (uint32_t t = 0; t < owner.size(); t++) {
      const uint32_t r = owner[t];
      if (r != kNoTable && (r >= n || !listed[r] || !known[r])) { drop(r); p.evicted.push_back(r); }
    }
    // the slot range becomes [0, new_max): kept tables at or above it move down into the lowest free slots below it
    const uint32_t old_max = max_tables;
    max_tables = new_max;
    if (owner.size() < new_max) owner.resize(new_max, kNoTable);
    free_slots.clear();
    for (uint32_t t = 0; t < new_max; t++) if (owner[t] == kNoTable) free_slots.insert(t);
    for (uint32_t t = new_max; t < std::max(old_max, (uint32_t)owner.size()); t++) {
      const uint32_t r = owner[t];
      if (r == kNoTable) continue;
      owner[t] = kNoTable;
      table[r] = kNoTable;
      const uint32_t to = take_free(r);  // cannot fail: at most new_max entries keep a table
      p.moves.push_back({r, t, to});
    }
    owner.resize(new_max);
    // the rest of the first max_tables get a slot
    for (size_t i = 0; i < keep; i++)
      if (table[cand[i]] == kNoTable && take_free(cand[i]) != kNoTable) p.admitted.push_back(cand[i]);
    return p;
  }
};

}  // namespace ibft
