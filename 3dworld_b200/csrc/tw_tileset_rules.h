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

} // namespace twts
