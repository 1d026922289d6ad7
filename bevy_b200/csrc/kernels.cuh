// kernels.cuh -- launchers of the sm_90a kernels (kernels.cu)
#pragma once
#include <cuda_runtime.h>
#include "device_types.cuh"

namespace b200vis {
void launch_propagate_cull(cudaStream_t st, const Rows &R, const Tile *tiles, uint32_t n_tiles, const CullViews &cvw,
                           const VisibleBufs &vb, DevStats *stats, uint32_t stages, uint32_t static_opt, uint32_t parity,
                           uint32_t *ticket = nullptr, uint32_t *ticket_base = nullptr, bool named_levels_only = false,
                           uint32_t rev = 0, uint8_t *gt_hint = nullptr);
// gt_hint (kernel 1b's PROPAGATE instantiations): one byte per tile of `tiles`, non-zero = stage all three old GlobalTransform
// rows, 0 = row 0 alone; the kernel rewrites it after every tile.  nullptr: always all three rows
void launch_propagate_cull_small(cudaStream_t st, const Rows &R, const Tile *tiles, uint32_t n_tiles, const CullViews &cvw,
                                 const VisibleBufs &vb, DevStats *stats, uint32_t stages, uint32_t static_opt, uint32_t parity);
unsigned long long kernel_launch_count();
// kernel 1b's instantiation for frames with pending external GlobalTransform marks (S_GT_EXT); stages must include PROPAGATE
void launch_propagate_cull_ext(cudaStream_t st, const Rows &R, const Tile *tiles, uint32_t n_tiles, const CullViews &cvw,
                               const VisibleBufs &vb, DevStats *stats, uint32_t stages, uint32_t static_opt, uint32_t parity,
                               uint32_t *ticket, uint32_t *ticket_base, uint32_t rev);
bool tile_kernel_is_default();   // B200VIS_TILE_KERNEL selects kernel 1b (unset, or tma)
bool tile_kernel_is_tma();
bool tile_kernel_is_warp();
bool tile_kernel_publishes_light_snapshot();
void launch_tile_warp(cudaStream_t st, const Rows &R, const WarpTile *tiles, const uint8_t *sched, uint32_t n_tiles, const CullViews &cvw,
                      const VisibleBufs &vb, DevStats *stats, uint32_t stages, uint32_t static_opt, uint32_t parity, uint32_t *counter);
// rev (kernel 1b and k_cull): 1 walks the tiles / rows in descending order, 0 ascending; the results do not depend on it
void launch_cull(cudaStream_t st, const Rows &R, const CullViews &cvw, const VisibleBufs &vb, DevStats *stats, uint32_t parity,
                 uint32_t rev);
// one group pass of a context with more than kMaxViews views: views view_base .. view_base + cvw.n_views - 1, merged into
// the ViewVisibility state the tile pass left (k_cull's MERGE instantiation)
void launch_cull_group(cudaStream_t st, const Rows &R, const CullViews &cvw, const VisibleBufs &vb, DevStats *stats, uint32_t parity,
                       uint32_t view_base, uint32_t rev);
void launch_mark_dirty_global(cudaStream_t st, const Rows &R);
void launch_expand_visible(cudaStream_t st, const VisibleBufs &vb, const DiffBufs &db, const uint32_t *row_of_rank, const FrameConsts *fc,
                           DevStats *stats, uint32_t parity, uint32_t n_rows, uint32_t max_views);
// b200vis_set_view_diff_sink: the per-class set algebra of views 0 .. slotted_views - 1 against their slots (vs), which must
// run before launch_expand_visible consumes the masks; then, anywhere behind it, the offsets of lists 0 .. n_views * 8
// and the ordered emit of the added / removed Entity lists
void launch_view_diff(cudaStream_t st, const VisibleBufs &vb, const ViewDiff &vd, const ViewSlots &vs, const uint32_t *row_of_rank,
                      const FrameConsts *fc, uint32_t parity, uint32_t slotted_views);
void launch_emit_view_diff(cudaStream_t st, const VisibleBufs &vb, const ViewDiff &vd, const ViewSlots &vs, uint32_t n_views,
                           uint32_t slotted_views);
// sink.entities != nullptr: also the Entity lists, offsets and active flags of b200vis_set_shadow_entities_sink;
// sd.added != nullptr: also the added / removed Entity lists and offsets of b200vis_set_shadow_diff_sink;
// kept_masks != nullptr: [n_lights * 6][words_stride], gets a copy of the run's mask bits before the expansion clears them;
// returns the copy's error (launch errors are left for cudaGetLastError)
cudaError_t launch_shadow_cull(cudaStream_t st, const Rows &R, const ShadowBufs &sb, const uint32_t *view_sets, uint32_t n_views,
                               uint32_t n_words, uint32_t n_chunks, uint32_t words_stride, uint32_t chunks_stride, DevStats *stats,
                               uint32_t changed_slot, const ShadowSink &sink, const ShadowDiff &sd, uint32_t *kept_masks);
// b200vis_emit_shadow_entities: the offsets, active flags and Entity lists of the last launch_shadow_cull into `sink`, expanded
// again from kept_masks and the chunk counts that run left; no select, no cull, no diff, the row lists untouched
cudaError_t launch_emit_shadow_entities(cudaStream_t st, const ShadowBufs &sb, const uint32_t *kept_masks, uint32_t n_rows, uint32_t n_words,
                                        uint32_t n_chunks, uint32_t words_stride, uint32_t chunks_stride, const uint32_t *row_of_rank,
                                        const ShadowSink &sink);
void launch_pack_cluster_bindings(cudaStream_t st, const FrameConsts *fc, const ClusterBufs &cb, const BindingBufs &bb, uint32_t max_views);
void launch_publish_visible_diff(cudaStream_t st, const VisibleBufs &vb, const DiffBufs &db, uint32_t *host_rows, uint32_t host_stride,
                                 uint32_t *host_counts, uint32_t n_views, uint32_t max_views);
void launch_cluster_assign(cudaStream_t st, const Rows &R, const Lights &L, const FrameConsts *fc, const ClusterBufs &cb,
                           DevStats *stats, uint32_t max_views);
bool cluster_fused_fits(uint32_t n_lights);
bool launch_cluster_fused(cudaStream_t st, const Rows &R, const Lights &L, const FrameConsts *fc, const ClusterBufs &cb,
                          DevStats *stats, uint32_t max_views);
void launch_publish_visible(cudaStream_t st, const VisibleBufs &vb, const DevStats *stats, uint32_t *host_rows, uint32_t host_stride,
                            uint32_t n_rows, uint32_t n_views, uint8_t *host_classes);
void launch_publish_clusters(cudaStream_t st, const FrameConsts *fc, const ClusterBufs &cb, uint32_t *host_offsets, uint32_t *host_indices,
                             uint32_t host_cap, const DevStats *stats, uint32_t *host_stats, uint32_t changed_slot, uint32_t frame, uint32_t max_views,
                             uint32_t *host_view_stats = nullptr);
void launch_tag_lights(cudaStream_t st, const Rows &R, const Lights &L, uint32_t *light_ord, uint32_t *all_tagged);
void launch_snapshot_lights(cudaStream_t st, const Rows &R, const Lights &L, float4 *snap);
void launch_writeback_columns(cudaStream_t st, const Rows &R, float *host_gt, uint32_t stride, uint32_t *host_gt_bits, uint8_t *host_vv,
                              uint32_t *host_vv_bits, uint8_t *vv_shadow);
void launch_writeback_tables(cudaStream_t st, const Rows &R, const TableBufs &tb, uint32_t which, uint32_t gt_tick, uint32_t vv_tick);
// b200vis_read_tables: which = B200VIS_RD_* bits, slots newer by Tick::is_newer_than(last_run, this_run)
void launch_read_tables(cudaStream_t st, const Rows &R, const TableBufs &tb, uint32_t which, uint32_t last_run, uint32_t this_run);
// b200vis_read_tables with RD_CULL_INPUTS: cull[t] = table t's cull inputs, fresh[entry] = read the slot in full (cleared);
// tab_caster[t] (nullptr = no table casters attached) = the caster byte a full read gives the slot's row;
// rr.tables (nullptr = no VisibilityRange columns attached) = the range columns a full read or a newer tick reads
void launch_read_table_cull(cudaStream_t st, const Rows &R, const TableBufs &tb, const DevTableCull *cull, uint8_t *fresh,
                            uint32_t last_run, uint32_t this_run, const uint8_t *tab_caster, uint8_t *caster, const RangeRead &rr);
// b200vis_writeback_tables with WB_SET_VISIBLE: set_visible() over the bytes the table slots hold, vv_shadow marked unknown
void launch_set_visible_tables(cudaStream_t st, const Rows &R, const TableBufs &tb, uint32_t vv_tick);
// b200vis_set_visible_entities_sink: counts = [max_views][chunks_stride][8] scratch, chunks_stride >= visible_entity_chunks(n_rows)
uint32_t visible_entity_chunks(uint32_t max_rows);
void launch_emit_visible_entities(cudaStream_t st, const VisibleBufs &vb, const uint32_t *rank, const uint64_t *keys, const FrameConsts *fc,
                                  const DevStats *stats, uint32_t n_rows, uint32_t max_views, uint32_t *counts, uint32_t chunks_stride,
                                  uint64_t *host_entities, uint32_t capacity, uint32_t *host_offsets);
// set_table_rows / set_tables / edit_topology: map[set[i].x] = set[i].y and fresh[set[i].x] = 1, then vv_shadow[reset[i]] = 0xFF
void launch_update_table_map(cudaStream_t st, uint32_t *map, const uint2 *set, uint32_t n_set, uint8_t *vv_shadow, const uint32_t *reset,
                             uint32_t n_reset, uint8_t *fresh);
void launch_record_push(cudaStream_t st, const uint32_t *block, uint32_t block_words, const ClusterBufs &cb);
void launch_slab_push(cudaStream_t st, const FrameConsts *fc, const ClusterBufs &cb, uint32_t *done, uint32_t max_views);
void launch_cluster_lists(cudaStream_t st, const FrameConsts *fc, const ClusterBufs &cb, DevStats *stats, uint32_t max_views);
void launch_unpack_trs(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, const float *src, int mark_only);
void launch_scatter_trs(cudaStream_t st, const Rows &R, uint32_t count, const uint32_t *rows, const float *src);
void launch_unpack_gt(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, const float *src);
void launch_write_gt_scattered(cudaStream_t st, const Rows &R, uint32_t count, const uint32_t *rows, const float *src);
void launch_clear_gt_ext(cudaStream_t st, const Rows &R, uint32_t n);
void launch_pack_gt(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, float *dst, uint32_t stride);
void launch_unpack_bounds(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, const float *bounds,
                          const uint8_t *flags, const uint8_t *cls, uint8_t *cls_col);
void launch_unpack_vv(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, const uint8_t *vv);
void launch_visibility_propagate(cudaStream_t st, const Rows &R, const Tile *tiles, uint32_t n_tiles, const uint8_t *vis, uint8_t *changed);
void launch_pack_inherited(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, const uint8_t *changed, uint8_t *out);
void launch_pack_ranges(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, uint32_t *out);
void launch_unpack_range_params(cudaStream_t st, float2 *se, uint8_t *ua, uint32_t first, uint32_t count, const float *src_se, const uint8_t *src_ua);
void launch_pack_state(cudaStream_t st, const Rows &R, uint32_t first, uint32_t count, uint8_t *out, uint32_t changed_bit);
// b200vis_edit_topology
void launch_rank_merge(cudaStream_t st, const uint64_t *old_keys, const uint32_t *old_row_of_rank, uint32_t n_old, const uint64_t *new_keys,
                       const uint32_t *new_rows, uint32_t n_new, uint64_t *keys, uint32_t *row_of_rank, uint32_t *rank, uint32_t *dup);
void launch_remap_rank_sets(cudaStream_t st, const uint32_t *old_sets, uint32_t *sets, uint32_t stride, uint32_t n_sets, uint32_t n_words,
                            uint32_t n_rows, uint32_t n_old_rows, const uint32_t *row_of_rank, const uint32_t *old_rank);
void launch_edit_rows(cudaStream_t st, const Rows &R, const RowEdit &e);
// b200vis_compact_topology
void launch_mark_listed_rows(cudaStream_t st, const RowLists &L, uint32_t max_count, uint8_t *mark, uint32_t n_rows);
void launch_mark_set_rows(cudaStream_t st, const uint32_t *sets, uint32_t stride, uint32_t n_sets, uint32_t n_words,
                          const uint32_t *row_of_rank, uint8_t *mark);
void launch_renumber_listed_rows(cudaStream_t st, const RowLists &L, uint32_t max_count, const uint32_t *old_to_new, uint32_t n_old);
void launch_gather_u32(cudaStream_t st, const uint32_t *src, const uint32_t *idx, uint32_t n, uint32_t *dst);
void launch_compact_ranks(cudaStream_t st, const uint32_t *old_row_of_rank, const uint64_t *old_keys, uint32_t n_old, const uint32_t *dropped,
                          uint32_t n_drop, const uint32_t *old_to_new, uint32_t *row_of_rank, uint32_t *rank, uint64_t *keys,
                          uint32_t *src_rank, uint32_t *not_identity);
void launch_permute_rows(cudaStream_t st, const RowPermute &p);
}
