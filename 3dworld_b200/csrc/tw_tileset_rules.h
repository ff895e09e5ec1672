// tw_tileset_rules.h - the cache rules of a tile set (tw_tileset.cu), host only and plain C++17 so that the tests can check them against a model.
// A tile (tx, ty) takes its incoming shadow rows from its neighbours TOWARD the light, (tx + sx, ty) and (tx, ty + sy) with sx = (lpos.x < 0 ? -1 : 1),
// sy = (lpos.y < 0 ? -1 : 1) (twi_shadow_plan_make). So its result depends on its own zvals and, transitively, on every resident tile upstream of it; the
// tiles DOWNSTREAM of it are (tx - sx, ty) and (tx, ty - sy). Invalidity is kept closed downstream: a valid tile never depends on an invalid one.
#pragma once
#include <stdint.h>
#include <map>
#include <utility>
#include <vector>

namespace twts {

typedef std::pair<int32_t, int32_t> key;           // (tx, ty)
typedef std::map<key, uint32_t> index_map;          // resident tile -> its slot in the set's slabs

inline int light_sign(float v) {return (v < 0.0f) ? -1 : 1;}

// Marks every resident tile reached from `seeds` by downstream steps invalid, the seeds included when resident. The walk stops at a tile that is not
// resident. valid is indexed by slab slot.
inline void invalidate_downstream(index_map const &where, std::vector<key> const &seeds, int sx, int sy, std::vector<uint8_t> &valid) {
	std::vector<uint8_t> seen(valid.size(), 0);
	std::vector<key> stack(seeds);
	while (!stack.empty()) {
		key const k = stack.back(); stack.pop_back();
		auto const it = where.find(k);
		if (it == where.end() || seen[it->second]) continue;
		seen[it->second] = 1; valid[it->second] = 0;
		stack.push_back(key(k.first - sx, k.second));
		stack.push_back(key(k.first, k.second - sy));
	}
}

// The tiles a relight recomputes for one light: the invalid requested tiles and their invalid resident upstream closure (each once, in walk order).
inline std::vector<key> recompute_batch(index_map const &where, std::vector<uint8_t> const &valid, std::vector<key> const &requested, int sx, int sy) {
	std::vector<uint8_t> seen(valid.size(), 0);
	std::vector<key> out, stack;
	for (key const &k : requested) {stack.push_back(k);}
	while (!stack.empty()) {
		key const k = stack.back(); stack.pop_back();
		auto const it = where.find(k);
		if (it == where.end() || seen[it->second] || valid[it->second]) continue;
		seen[it->second] = 1;
		out.push_back(k);
		stack.push_back(key(k.first + sx, k.second));
		stack.push_back(key(k.first, k.second + sy));
	}
	return out;
}

// The host side of a set that put and remove change: residency, slab slots and each light slot's valid bits. A frame launch
// (tw_tile_set_create_tiles_launch) applies its removes and puts to a copy, plans its relight against the copy and commits it.
struct state {
	index_map where;                                 // resident tile -> slab slot
	std::vector<uint32_t> free_slots;                // slots of removed tiles, reused first (the last freed first)
	uint32_t used = 0;                               // slots handed out so far
	std::vector<std::vector<uint8_t>> valid;         // per light slot, indexed by slab slot (at least `used` entries)
};
struct signs {int sx, sy;};                          // a light slot's (sx, sy): from its params, or (1, 1) before it has any

// Removes resident keys (each named once, checked by the caller): the slots are freed and invalid, and the tiles downstream of each lose an incoming row.
inline void remove_tiles(state &s, std::vector<key> const &keys, std::vector<signs> const &sg) {
	for (key const &k : keys) {
		uint32_t const slot = s.where[k];
		s.where.erase(k);
		s.free_slots.push_back(slot);
		for (std::vector<uint8_t> &v : s.valid) {v[slot] = 0;}
	}
	for (size_t l = 0; l < s.valid.size(); ++l) {
		std::vector<key> seeds;
		for (key const &k : keys) {seeds.push_back(key(k.first - sg[l].sx, k.second)); seeds.push_back(key(k.first, k.second - sg[l].sy));}
		invalidate_downstream(s.where, seeds, sg[l].sx, sg[l].sy, s.valid[l]);
	}
}

// The slab slot of each put key (named once): a resident tile keeps its own, new tiles take freed slots first, then fresh ones. Returns the new `used`.
inline uint32_t put_slots(state const &s, std::vector<key> const &keys, std::vector<uint32_t> &free_left, std::vector<int> &idx) {
	free_left = s.free_slots;
	uint32_t next = s.used;
	idx.resize(keys.size());
	for (size_t i = 0; i < keys.size(); ++i) {
		auto const it = s.where.find(keys[i]);
		if (it != s.where.end()) {idx[i] = (int)it->second;}
		else if (!free_left.empty()) {idx[i] = (int)free_left.back(); free_left.pop_back();}
		else {idx[i] = (int)next++;}
	}
	return next;
}

// Commits a put with the slots of put_slots: the tiles are resident, and each put tile and its downstream closure are invalid in every light slot.
inline void put_tiles(state &s, std::vector<key> const &keys, std::vector<int> const &idx, std::vector<uint32_t> &free_left, uint32_t used, std::vector<signs> const &sg) {
	for (size_t i = 0; i < keys.size(); ++i) {s.where.emplace(keys[i], (uint32_t)idx[i]);}
	s.free_slots.swap(free_left); s.used = used;
	for (size_t l = 0; l < s.valid.size(); ++l) {
		if (s.valid[l].size() < used) s.valid[l].resize(used, 0);
		invalidate_downstream(s.where, keys, sg[l].sx, sg[l].sy, s.valid[l]);
	}
}

// What tw_tile_set_stale lists: the resident tiles, in (x, y) order, that are invalid in one of the first reset.size() light slots, or every resident tile when
// one of those slots is reset (its params differ from the request's or it has none).
inline std::vector<key> stale_tiles(state const &s, std::vector<uint8_t> const &reset) {
	std::vector<key> out;
	for (auto const &kv : s.where) { // a relight of every resident tile recomputes exactly the invalid ones (their upstream closure is invalid too)
		bool stale = false;
		for (size_t l = 0; l < reset.size() && !stale; ++l) {stale = reset[l] || !s.valid[l][kv.second];}
		if (stale) out.push_back(kv.first);
	}
	return out;
}

// tw_tile_set_stale_after: the stale tiles once `removed` (resident) and then `put` have been applied to a copy of s.
inline std::vector<key> stale_after(state s, std::vector<key> const &removed, std::vector<key> const &put, std::vector<signs> const &sg, std::vector<uint8_t> const &reset) {
	if (!removed.empty()) remove_tiles(s, removed, sg);
	if (!put.empty()) {
		std::vector<uint32_t> free_left;
		std::vector<int> idx;
		uint32_t const used = put_slots(s, put, free_left, idx);
		put_tiles(s, put, idx, free_left, used, sg);
	}
	return stale_tiles(s, reset);
}

} // namespace twts
