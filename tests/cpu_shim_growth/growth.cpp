/*
 * tests/cpu_shim_growth/growth.cpp — TEST-ONLY host build of the map growth (lv_map.cu map_grow).
 *
 * The CPU shim (tests/cpu_shim/shim.cpp) compiled as it is, plus the growth of its map: fresh tables at the shim's ratios,
 * every old slot re-inserted by the product's voxel_rehash_item / block_rehash_item (lv_voxel_map.h, the functions the
 * rehash kernel runs), the used prefix of the arena copied with its indices unchanged.  Like the shim it is not part of the
 * product and is not reachable from the C ABI.
 */
#include "../cpu_shim/shim.cpp"

extern "C" {

/* grow to the shim's ratios for `cap` points: 8 table slots and 64 arena entries per point (shim_map_create_cap) */
void shim_map_grow(ShimMap* sm, int64_t cap) {
    uint32_t slots = 1u << 14;
    while (slots < 8 * (uint64_t)(cap + 65536)) slots <<= 1;
    uint4 empty; empty.x = empty.y = 0xFFFFFFFFu; empty.z = empty.w = 0;
    uint4 zero; zero.x = zero.y = zero.z = zero.w = 0;
    std::vector<uint4> table(2 * (size_t)slots, zero), btable(slots / 4, empty);
    for (uint32_t s = 0; s < slots; ++s) table[2 * (size_t)s] = empty;
    std::vector<float4> arena((size_t)64 * (size_t)(cap + 65536) + (1u << 20));
    if (arena.size() < sm->arena.size()) arena.resize(sm->arena.size());
    const uint32_t top = std::min<uint32_t>(sm->counters[kCtrArenaTop], (uint32_t)sm->arena.size());
    std::copy(sm->arena.begin(), sm->arena.begin() + top, arena.begin());
    VoxelMapRW r = sm->rw;
    r.table = table.data(); r.mask = slots - 1; r.btable = btable.data(); r.bmask = slots / 4 - 1;
    r.arena = arena.data(); r.arena_cap = (uint32_t)arena.size();
    sm->counters[kCtrSlotsUsed] = 0;
    sm->counters[kCtrBlocksUsed] = 0;
    for (uint32_t s = 0; s <= sm->rw.mask; ++s) voxel_rehash_item(r, sm->table.data(), s);
    for (uint32_t s = 0; s <= sm->rw.bmask; ++s) block_rehash_item(r, sm->btable.data(), s);
    sm->table.swap(table);              /* the buffers move with the swap: r's pointers stay valid */
    sm->btable.swap(btable);
    sm->arena.swap(arena);
    sm->touched.assign(slots, 0u);
    sm->dirty.assign(slots, 0u);
    r.touched = sm->touched.data(); r.dirty = sm->dirty.data(); r.list_cap = slots;
    sm->rw = r;
    sm->view = map_view_of(r);
}
/* one device counter of the map (lv_voxel_map.h kCtr*) */
uint32_t shim_map_counter(const ShimMap* sm, int k) { return sm->counters[k]; }

}  // extern "C"
