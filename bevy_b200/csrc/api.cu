// api.cu -- host runtime + C ABI of libb200vis.so (include/b200vis.h).
//
// Owns the SoA device mirror of the ECS columns, the execution plan built from the hierarchy
// (tiles and passes), the per-frame constants, and the stream every stage is issued on.
// There is NO CPU fallback: without a CUDA device b200vis_create fails with B200VIS_ERR_CUDA.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

#include <chrono>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>

#include "../../include/b200vis.h"
#include "device_types.cuh"
#include "host_view.hpp"
#include "kernels.cuh"

using namespace b200vis;

static thread_local std::string g_create_error;

// ---- NCCL through dlopen: no link-time dependency, and the process keeps ONE NCCL (the one torch already loaded) ----
namespace {
struct NcclId { char b[128]; };   // ncclUniqueId (passed BY VALUE to ncclCommInitRank)
struct NcclApi {
    using Id = NcclId;
    void *lib = nullptr;
    int (*GetUniqueId)(void *) = nullptr;
    int (*CommInitRank)(void **, int, NcclId, int) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    bool load() {
        if (lib) return true;
        lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) return false;
        GetUniqueId = reinterpret_cast<decltype(GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
        CommInitRank = reinterpret_cast<decltype(CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
        AllGather = reinterpret_cast<decltype(AllGather)>(dlsym(lib, "ncclAllGather"));
        CommDestroy = reinterpret_cast<decltype(CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
        GetErrorString = reinterpret_cast<decltype(GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
        return GetUniqueId && CommInitRank && AllGather && CommDestroy && GetErrorString;
    }
};
NcclApi g_nccl;
constexpr int kNcclUint32 = 3;   // ncclUint32 in nccl.h's ncclDataType_t
}

struct Plan;
static void free_plan(Plan *p);

struct b200vis_ctx {
    b200vis_config cfg{};
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    // Frame pipelining: the latency-bound tail of frame f (visible-list expansion, cluster kernels) runs on a side
    // stream while frame f+1's tile pass already runs on the main stream (masks / counters / constants are
    // double or triple buffered by frame number).
    cudaStream_t side_stream = nullptr;
    cudaStream_t clus_stream = nullptr; cudaEvent_t ev_clus = nullptr;   // pipelined frames: the cluster branch of the tail (exchange -> cluster kernel) runs beside the list expansion
    cudaEvent_t ev_tile = nullptr, ev_side[3] = {nullptr, nullptr, nullptr}, ev_expand[2] = {nullptr, nullptr}, ev_pub = nullptr;
    bool pub_pending = false;           // a publish_visible copy is in flight on the side stream
    bool pipeline = true, side_pending = false;
    // a frame whose tail was started (expand + cluster assign on the side stream) but whose CLUSTER_LISTS stage is
    // still to come in a later b200vis_run call (multi-GPU: the host all-gathers the slabs in between)
    bool tail_open = false; uint32_t open_frame = 0; const FrameConsts *open_fc = nullptr;
    // light blocks [3 frame slots]: float4 snap[cap32] | float range[cap32] | uint64 layers[cap32] (cap32 = cl.max_lights).  The
    // snap part is what the tile pass fills per frame; with several GPUs the whole block is what one all-gather exchanges
    uint8_t *d_lrec = nullptr, *d_lrec_all = nullptr; size_t lrec_bytes = 0;
    float4 *light_snap_slot(uint32_t slot) const { return reinterpret_cast<float4 *>(d_lrec + (size_t)slot * lrec_bytes); }
    uint32_t *d_tag_flag = nullptr;     // 1 if every light row carries its ordinal (k_tag_lights)
    uint32_t *d_light_ord = nullptr;    // [max_entities] light ordinal per row, 0xFFFFFFFF = not a light (rewritten on set_lights)
    bool lights_tag_dirty = true, lights_tagged = false;
    std::string err;

    uint32_t n = 0;                 // current row count
    Rows rows{};                    // device SoA (capacity cfg.max_entities)
    uint64_t *d_layers_ext = nullptr; bool have_layers_ext = false; uint64_t view_layers_ext[kMaxCameras][3] = {};   // RenderLayers blocks 1..3
    uint32_t *d_parent = nullptr; uint64_t *d_layers = nullptr; uint32_t *d_range = nullptr;
    uint32_t *d_rank = nullptr, *d_row_of_rank = nullptr; uint8_t *d_dirty = nullptr;
    bool have_layers = false, have_range = false, rank_identity = true, topology_set = false;
    bool bounds_set = false;

    // plan
    Tile *d_tiles = nullptr; uint32_t tiles_cap = 0;
    WarpTile *d_wtiles = nullptr; uint8_t *d_sched = nullptr; uint32_t *d_wtopo = nullptr;   // k_tile_warp's view of the plan
    uint32_t *d_tile_counter = nullptr;
    uint32_t *d_tile_ticket = nullptr; uint32_t tile_ticket_base = 0;   // dynamic tile hand-out of the default kernel: never reset, the host tracks the base
    // kernel 1b's staging hint, one byte per tile descriptor (indexed like d_tiles): non-zero = stage all three old
    // GlobalTransform rows, 0 = row 0 alone (tile_kernel_1b.cuh).  Every new plan starts at all three; any value is correct.
    uint8_t *d_tile_hint = nullptr; uint32_t hint_cap = 0;
    bool gt_stage_full = false;     // B200VIS_GT_STAGE=full (experiment switch, read at create): always stage all three rows
    // Full-world sweeps launched so far: every kernel 1b launch over a pass and every k_cull launch counts one.  Each sweep
    // walks the rows opposite to the previous one (next_sweep_reversed), so it starts on the rows the previous sweep touched
    // last, which are the ones still in L2.  Any order gives the same results; only the parity matters.
    uint32_t sweep_count = 0;
    std::vector<uint32_t> pass_begin;   // tile index ranges per pass: [pass_begin[p], pass_begin[p+1])
    std::vector<uint32_t> pass_small;   // the first pass_small[p] tiles of pass p have <= 32 rows (B200VIS_SPLIT_DEEP_TILES)
    std::vector<uint8_t> pass_named;    // every tile of pass p is flat or walks with named level barriers (Tile::lvl_warps): the tile kernel may let a CTA's warps drift a tile apart
    int static_opt = 1;
    // b200vis_write_global_transforms_scattered left S_GT_EXT marks that no run with PROPAGATE has consumed yet (rows the
    // edit despawned since may have lost theirs): the next propagate pass runs kernel 1b's marked instantiation
    bool gt_ext_pending = false;
    // b200vis_edit_topology: the host plan kept between calls, the world's keys (Entity::to_bits()) in rank order -- on the
    // host after set_topology, on the device from the first edit that needs a merge -- and the spare rank arrays a merge
    // writes into (swapped in when the edit is committed)
    Plan *hplan = nullptr;
    std::vector<uint64_t> h_keys; bool keys_resident = false; uint64_t max_key = 0;
    uint64_t *d_keys = nullptr, *d_keys2 = nullptr; uint32_t *d_rank2 = nullptr, *d_row_of_rank2 = nullptr;
    uint8_t *h_edit = nullptr; size_t h_edit_bytes = 0; cudaEvent_t ev_edit = nullptr;   // pinned staging of an edit's uploads

    // per-frame constants
    // The "frame blob": FrameConsts followed by the packed per-view plane tables and z thresholds.
    // Setters edit the host working copy; run() packs it into the next pinned ring slot and issues
    // ONE async H2D copy, so per-frame constant updates never block on the stream.
    FrameConsts consts{};               // host working copy
    std::vector<float> tab_x[kMaxCameras], tab_y[kMaxCameras], tab_z[kMaxCameras], tab_thr[kMaxCameras];
    static constexpr int kRing = 4;
    uint8_t *h_ring[kRing] = {nullptr, nullptr, nullptr, nullptr};   // pinned
    cudaEvent_t ring_ev[kRing] = {nullptr, nullptr, nullptr, nullptr};
    int ring_next = 0;
    size_t blob_cap = 0;
    uint8_t *d_blob2[3] = {nullptr, nullptr, nullptr};   // live-mode device blobs, slot = frame % 3
    uint8_t *d_blob = nullptr;          // the one the current frame uses
    FrameConsts *d_consts = nullptr;    // == d_blob
    bool consts_dirty = true;
    const uint8_t *blob_flushed = nullptr;   // the device blob the last flush wrote (the only one known to be current)
    size_t blob_used = 0;               // bytes of the last packed blob
    struct Recorded { FrameConsts host; uint8_t *dev; size_t bytes; };
    std::vector<Recorded> recorded;     // b200vis_record_frame_constants
    int replay_slot = -1;               // >= 0: b200vis_run reads recorded[replay_slot] instead of the live copy
    // optional per-stage timing (b200vis_set_profiling)
    bool profiling = false;
    static constexpr int kProfFrames = 256;
    cudaEvent_t (*prof_ev)[6] = nullptr;   // [kProfFrames][6]: main 0,1 (tile); side 2,3,4 (expand, cluster); created on first use
    int prof_count = 0;

    // visible set
    VisibleBufs vis{};
    DiffBufs diff{}; bool diff_on = false;      // SURVEY 8(f) N1 (b200vis_enable_visible_diff)
    uint32_t *diff_sink_rows_d = nullptr, *diff_sink_counts_d = nullptr; uint32_t diff_sink_cap = 0;
    BindingBufs bind{}; uint32_t *d_bind_map = nullptr; uint32_t bind_map_cap = 0;   // SURVEY 8(f) N2 (b200vis_set_cluster_bindings)
    // SURVEY 8(f) N3: shadow-view culling (b200vis_set_shadow_lights / b200vis_run_shadow_culling)
    ShadowBufs shadow{}; ShadowLight *d_shadow_lights = nullptr; uint8_t *d_caster = nullptr;
    uint32_t shadow_cap_lights = 0, shadow_cap_list = 0; std::vector<ShadowLight> h_shadow;
    // SURVEY 8(f) N4: VisibilityRange columns + range views; Visibility column + the rows the last propagate wrote
    float2 *d_range_se = nullptr; uint8_t *d_range_ua = nullptr; float4 *d_range_views = nullptr; uint32_t n_range_views = 0;
    uint8_t *d_visibility = nullptr, *d_iv_changed = nullptr; bool iv_ran = false;
    DevStats *d_stats = nullptr; DevStats *h_stats = nullptr;   // h pinned
    uint32_t frame = 0, parity = 0;

    // lights + clusters
    std::vector<uint32_t> h_light_row; std::vector<float> h_light_range;   // host copies (b200vis_set_shadow_lights resolves ordinals)
    Lights lights{}; uint32_t *d_light_row = nullptr; float *d_light_range = nullptr; uint64_t *d_light_layers = nullptr;
    // RenderLayers blocks 1..3 of the lights (by ordinal) and of the shadow items (by item), allocated on first use; *_ext_on:
    // some entry is nonzero (b200vis_set_light_render_layers_ext / b200vis_set_shadow_item_render_layers_ext)
    uint64_t *d_light_layers_ext = nullptr; bool light_ext_on = false;
    uint64_t *d_shadow_layers_ext = nullptr; uint32_t shadow_ext_cap = 0; bool shadow_ext_on = false;
    ClusterBufs cl{}; uint32_t *d_slab = nullptr; void *ext_send = nullptr, *ext_recv = nullptr;
    size_t slab_bytes = 0;

    // result sink (mapped pinned host memory written by publish kernels)
    b200vis_result_sink sink{}; bool have_sink = false;
    uint32_t *sink_rows_d = nullptr, *sink_off_d = nullptr, *sink_idx_d = nullptr, *sink_stats_d = nullptr;
    uint8_t *sink_cls_d = nullptr; uint8_t *d_cls = nullptr;   // VisibilityClass masks: sink alias, per-row column
    uint32_t *view_stats_sink = nullptr, *view_stats_d = nullptr;   // b200vis_set_view_stats_sink: [max_views][4], host and device alias
    // b200vis_set_visible_entities_sink: device aliases, and the per (view, chunk, class) counts of the emit
    uint64_t *ent_sink_d = nullptr; uint32_t *ent_off_d = nullptr; uint32_t ent_cap = 0;
    uint32_t *d_ent_counts = nullptr; uint32_t ent_chunks = 0;
    // b200vis_set_shadow_entities_sink: device aliases (entities == nullptr: none), its max_items, and the device offsets
    ShadowSink shsink{}; uint32_t shsink_max_items = 0; uint32_t *d_shadow_off = nullptr; size_t shadow_off_cap = 0;
    // b200vis_emit_shadow_entities: the last run's mask bits (copied while an entity sink is registered), and whether they
    // still describe the installed items over the current rows (cleared by new items and by every topology change)
    uint32_t *d_shadow_kept = nullptr; size_t shadow_kept_cap = 0; bool shadow_emit_ready = false;
    // b200vis_set_shadow_diff_sink: the device state (added == nullptr: none) and the host's side of it: max_items / max_slots,
    // the installed items' slots, and which slots may hold entries (the ones a run named since they were last emptied)
    ShadowDiff sdiff{}; uint32_t sdiff_max_items = 0, sdiff_max_slots = 0;
    std::vector<uint32_t> h_sdiff_slot; std::vector<uint8_t> sdiff_held;
    // b200vis_set_view_diff_sink: the device state (added == nullptr: none), max_slots, the view -> slot map of
    // b200vis_set_view_diff_slots ([max_views], kNoDiffSlot = none), and which slots may hold entries
    ViewDiff vdiff{}; uint32_t vdiff_max_slots = 0;
    std::vector<uint32_t> h_vdiff_slot; std::vector<uint8_t> vdiff_held;

    b200vis_column_sinks colsink{}; bool have_colsink = false;          // b200vis_set_column_sinks (device aliases below)
    float *col_gt_d = nullptr; uint32_t *col_gt_bits_d = nullptr, *col_vv_bits_d = nullptr; uint8_t *col_vv_d = nullptr;
    uint8_t *d_vv_shadow = nullptr;     // what the host ViewVisibility column holds (0xFF = unknown)
    bool gt_aos_valid = false;
    bool step_defers_stats = false;     // inside b200vis_step: the CULL run leaves the sink's stats block to the CLUSTER run
    float *d_gt_aos = nullptr;          // dense write-back: the GlobalTransform column in the host's layout, copied by the DMA engine
    uint32_t last_gt_changed = 0;       // Changed<GlobalTransform> rows of the last frame whose statistics the host has seen
    // b200vis_set_tables: the registry, the host copy of the slot -> row maps (every table's map back to back, as on the
    // device) and its inverse, and the host-memory registrations the library owns
    bool tables_set = false;
    std::vector<b200vis_table> h_tabs; std::vector<uint32_t> tab_off;   // tab_off[t] = table t's first map entry
    std::vector<b200vis_table_inputs> h_tab_in; b200vis_transform_layout tab_layout{};   // b200vis_set_tables_ex's input columns
    std::vector<uint32_t> h_tab_map, row_slot;                           // row_slot[row] = the row's map entry, or kNoParent
    std::vector<std::pair<uintptr_t, size_t>> host_regs;
    DevTable *d_tabs = nullptr; uint32_t *d_tab_chunks = nullptr; uint32_t tab_chunks_cap = 0, n_tab_chunks = 0;
    uint32_t *d_tab_map = nullptr; size_t tab_map_cap = 0; uint32_t *d_tab_total = nullptr;
    uint8_t *d_tvv_shadow = nullptr;    // per row: the ViewVisibility byte the row's table slot holds (0xFF = unknown)
    uint8_t *d_tab_upd = nullptr; size_t tab_upd_cap = 0;   // map updates on their way to k_update_table_map
    std::vector<uint32_t> pend_touched, pend_reset;          // queued map entries / shadow resets, sent by flush_table_updates
    uint8_t *h_tab_stage = nullptr; size_t h_tab_stage_cap = 0; cudaEvent_t ev_tab = nullptr;   // pinned staging of a batch
    // b200vis_set_table_cull_inputs: the entries of the last call (kept across b200vis_set_tables, which only detaches them),
    // whether they are attached, their device form, and per map entry the "read in full" mark k_read_table_cull clears
    std::vector<b200vis_table_cull_inputs> h_tab_cull; b200vis_bounds_layout cull_layout{}; bool cull_attached = false;
    DevTableCull *d_tab_cull = nullptr; uint8_t *d_tab_fresh = nullptr;
    // b200vis_set_table_shadow_casters: the attached per-table caster bytes, and their device copy
    std::vector<uint8_t> h_tab_caster; bool caster_attached = false; uint8_t *d_tab_caster = nullptr;
    // b200vis_set_table_visibility_ranges: the last attached entries (a table that stays keeps its entry across set_tables,
    // so its columns stay registered and it is not read in full when attached again unchanged; empty = none attached),
    // whether some table's are read, their layout, and their device form
    std::vector<b200vis_table_visibility_ranges> h_tab_range; b200vis_visibility_range_layout range_layout{};
    bool range_attached = false; DevTableRange *d_tab_range = nullptr;
    bool cull_fresh_pending = false;    // slots (re)mapped or tables (re)attached since the last RD_CULL_INPUTS read
    double step_t[6] = {0, 0, 0, 0, 0, 0}; uint64_t step_n = 0;   // B200VIS_STEP_TRACE: host time per phase of b200vis_step
    void *nccl_comm = nullptr;          // b200vis_comm_init
    uint32_t *d_gather = nullptr;       // [world][slab] when the library owns the exchange
    // peer-memory exchange (b200vis_p2p_export / _import): [2][world][slab] + flags [2][world], mapped into every rank
    uint32_t *d_xbuf = nullptr; size_t xbuf_flag_offset = 0; void *peer_map[8] = {}; bool peer_ipc[8] = {}; bool p2p_ready = false;
    uint32_t *d_push_done = nullptr;
    b200vis_cluster_feedback auto_fb[kMaxCameras]{};   // b200vis_step: last frame's Clusters feedback

    // staging for AoS <-> SoA conversion
    uint8_t *d_stage = nullptr; size_t stage_bytes = 0;
    uint8_t *h_stage = nullptr;         // pinned, same size (downloads)
};

static int32_t fail(b200vis_ctx *c, int32_t code, const char *fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    if (c) c->err = buf; else g_create_error = buf;
    return code;
}
#define CU(call)                                                                                        \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess)                                                                          \
            return fail(ctx, e_ == cudaErrorMemoryAllocation ? B200VIS_ERR_OUT_OF_MEMORY : B200VIS_ERR_CUDA, \
                        "%s failed: %s", #call, cudaGetErrorString(e_));                                \
    } while (0)

template <typename T>
static cudaError_t dalloc(T **p, size_t count) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(p), std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) e = cudaMemset(*p, 0, std::max<size_t>(count, 1) * sizeof(T));
    return e;
}

extern "C" int32_t b200vis_abi_version(void) { return B200VIS_ABI_VERSION; }
extern "C" uint64_t b200vis_kernel_launch_count(void) { return kernel_launch_count(); }
extern "C" void b200vis_struct_sizes(uint32_t out[6]) {
    out[0] = sizeof(b200vis_config); out[1] = sizeof(b200vis_view); out[2] = sizeof(b200vis_cluster_view);
    out[3] = sizeof(b200vis_frame_stats); out[4] = sizeof(b200vis_cluster_config); out[5] = sizeof(b200vis_cluster_feedback);
}

extern "C" const char *b200vis_last_error(const b200vis_ctx *ctx) {
    return ctx ? ctx->err.c_str() : g_create_error.c_str();
}

extern "C" void b200vis_destroy(b200vis_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    Rows &r = ctx->rows;
    void *dev[] = {r.trsA, r.trsB, r.trsC, r.gt0, r.gt1, r.gt2, r.bndA, r.bndB, r.flags, r.state, r.topo,
                   ctx->d_parent, ctx->d_layers, ctx->d_range, ctx->d_rank, ctx->d_row_of_rank, ctx->d_dirty,
                   ctx->d_layers_ext, ctx->d_vv_shadow, ctx->d_gt_aos, ctx->d_tiles, ctx->d_wtiles, ctx->d_sched, ctx->d_wtopo, ctx->d_tile_counter, ctx->d_tile_ticket, ctx->d_tile_hint, ctx->d_blob2[0], ctx->d_blob2[1], ctx->d_blob2[2], ctx->d_lrec, ctx->d_lrec_all, ctx->d_tag_flag, ctx->d_light_ord,
                   ctx->vis.mask, ctx->vis.chunk_count, ctx->vis.lists, ctx->vis.classes, ctx->d_cls, ctx->d_stats, ctx->d_light_row,
                   ctx->d_light_range, ctx->d_light_layers, ctx->d_slab, ctx->cl.offsets, ctx->cl.indices, ctx->d_stage,
                   ctx->diff.prev, ctx->diff.words, ctx->diff.chunk, ctx->diff.lists, ctx->diff.count,
                   ctx->bind.oc, ctx->bind.il, ctx->bind.count, ctx->d_bind_map,
                   ctx->d_range_se, ctx->d_range_ua, ctx->d_range_views, ctx->d_visibility, ctx->d_iv_changed,
                   ctx->d_shadow_lights, ctx->d_caster, ctx->shadow.mask, ctx->shadow.chunk_count, ctx->shadow.lists,
                   ctx->shadow.count, ctx->shadow.active, ctx->d_keys, ctx->d_keys2, ctx->d_rank2, ctx->d_row_of_rank2,
                   ctx->d_tabs, ctx->d_tab_chunks, ctx->d_tab_map, ctx->d_tab_total, ctx->d_tvv_shadow, ctx->d_tab_upd,
                   ctx->d_tab_cull, ctx->d_tab_fresh, ctx->d_ent_counts, ctx->d_shadow_off, ctx->d_tab_caster,
                   ctx->d_tab_range, const_cast<uint32_t *>(ctx->sdiff.slot), ctx->sdiff.prev, ctx->sdiff.prev_count,
                   ctx->sdiff.words, ctx->sdiff.chunk, ctx->sdiff.dev_offsets, ctx->vdiff.prev, ctx->vdiff.prev_count,
                   ctx->vdiff.words, ctx->vdiff.chunk, ctx->vdiff.dev_offsets, ctx->d_light_layers_ext, ctx->d_shadow_layers_ext,
                   ctx->d_shadow_kept};
    for (void *p : dev) if (p) cudaFree(p);
    for (const auto &r : ctx->host_regs) cudaHostUnregister(reinterpret_cast<void *>(r.first));
    cudaGetLastError();
    if (ctx->h_tab_stage) cudaFreeHost(ctx->h_tab_stage);
    if (ctx->ev_tab) cudaEventDestroy(ctx->ev_tab);
    if (ctx->h_edit) cudaFreeHost(ctx->h_edit);
    if (ctx->ev_edit) cudaEventDestroy(ctx->ev_edit);
    free_plan(ctx->hplan);
    for (int i = 0; i < b200vis_ctx::kRing; ++i) {
        if (ctx->h_ring[i]) cudaFreeHost(ctx->h_ring[i]);
        if (ctx->ring_ev[i]) cudaEventDestroy(ctx->ring_ev[i]);
    }
    if (ctx->prof_ev) {
        for (int i = 0; i < b200vis_ctx::kProfFrames; ++i) for (cudaEvent_t e : ctx->prof_ev[i]) if (e) cudaEventDestroy(e);
        delete[] ctx->prof_ev;
    }
    if (ctx->h_stats) cudaFreeHost(ctx->h_stats);
    if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
    if (ctx->step_n && getenv("B200VIS_STEP_TRACE"))
        fprintf(stderr, "[b200vis_step] %llu steps, host us/step: upload %.1f  frusta %.1f  run(prop|cull) %.1f  cluster prologue %.1f  run(cluster) %.1f  wait %.1f\n",
                (unsigned long long)ctx->step_n, 1e6 * ctx->step_t[0] / ctx->step_n, 1e6 * ctx->step_t[1] / ctx->step_n, 1e6 * ctx->step_t[2] / ctx->step_n,
                1e6 * ctx->step_t[3] / ctx->step_n, 1e6 * ctx->step_t[4] / ctx->step_n, 1e6 * ctx->step_t[5] / ctx->step_n);
    if (ctx->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->nccl_comm);
    if (ctx->d_gather) cudaFree(ctx->d_gather);
    for (uint32_t r = 0; r < 8; ++r) if (ctx->peer_map[r] && r != ctx->cl.rank && ctx->peer_ipc[r]) cudaIpcCloseMemHandle(ctx->peer_map[r]);
    if (ctx->d_xbuf) cudaFree(ctx->d_xbuf);
    if (ctx->d_push_done) cudaFree(ctx->d_push_done);
    for (auto &r : ctx->recorded) if (r.dev) cudaFree(r.dev);
    if (ctx->side_stream) { cudaStreamSynchronize(ctx->side_stream); cudaStreamDestroy(ctx->side_stream); }
    if (ctx->clus_stream) { cudaStreamSynchronize(ctx->clus_stream); cudaStreamDestroy(ctx->clus_stream); }
    if (ctx->ev_clus) cudaEventDestroy(ctx->ev_clus);
    if (ctx->ev_tile) cudaEventDestroy(ctx->ev_tile);
    if (ctx->ev_pub) cudaEventDestroy(ctx->ev_pub);
    for (cudaEvent_t e : ctx->ev_side) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ctx->ev_expand) if (e) cudaEventDestroy(e);
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    delete ctx;
}

extern "C" int32_t b200vis_create(const b200vis_config *cfg, b200vis_ctx **out) {
    b200vis_ctx *ctx = nullptr;   // for CU(): errors before allocation go to the thread-local slot
    if (!cfg || !out) return fail(nullptr, B200VIS_ERR_INVALID_ARG, "b200vis_create: null argument");
    *out = nullptr;
    if (cfg->max_views == 0 || cfg->max_views > B200VIS_MAX_CAMERAS)
        return fail(nullptr, B200VIS_ERR_INVALID_ARG, "max_views must be in 1..%u", B200VIS_MAX_CAMERAS);
    // the cluster exchange (slab trailer, light records) and its tests cover eight views per rank
    if (cfg->world_size > 1 && cfg->max_views > B200VIS_MAX_VIEWS)
        return fail(nullptr, B200VIS_ERR_INVALID_ARG, "max_views > %u needs world_size 1", B200VIS_MAX_VIEWS);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, B200VIS_ERR_CUDA, "no CUDA device (%s): libb200vis has no CPU fallback",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, B200VIS_ERR_INVALID_ARG, "device %d out of range", cfg->device);
    CU(cudaSetDevice(cfg->device));
    ctx = new b200vis_ctx();
    ctx->cfg = *cfg;
    ctx->device = cfg->device;
    if (ctx->cfg.world_size == 0) ctx->cfg.world_size = 1;
    if (ctx->cfg.max_cluster_indices == 0) ctx->cfg.max_cluster_indices = 1u << 20;
    const size_t N = cfg->max_entities, V = cfg->max_views;
    int32_t rc = [&]() -> int32_t {
        CU(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
        ctx->stream = ctx->own_stream;
        Rows &r = ctx->rows;
        const size_t NP = N + 32;   // the TMA-staged tile kernel copies 16-row aligned windows: pad every staged column
        CU(dalloc(&r.trsA, NP)); CU(dalloc(&r.trsB, NP)); CU(dalloc(&r.trsC, NP));
        CU(dalloc(&r.gt0, NP)); CU(dalloc(&r.gt1, NP)); CU(dalloc(&r.gt2, NP));
        CU(dalloc(&r.bndA, NP)); CU(dalloc(&r.bndB, NP));
        CU(dalloc(&r.flags, NP)); CU(dalloc(&r.state, NP)); CU(dalloc(&r.topo, NP));
        CU(dalloc(&ctx->d_parent, N)); CU(dalloc(&ctx->d_layers, N)); CU(dalloc(&ctx->d_range, N));
        CU(dalloc(&ctx->d_rank, N)); CU(dalloc(&ctx->d_row_of_rank, N)); CU(dalloc(&ctx->d_dirty, N));
        r.parent = ctx->d_parent;
        ctx->tiles_cap = (uint32_t)(N / 1 + 1);   // worst case one tile per row is never reached; see planner
        ctx->tiles_cap = (uint32_t)std::min<size_t>(N + 1, (N / 8) + 1024);
        CU(dalloc(&ctx->d_tiles, ctx->tiles_cap));
        CU(dalloc(&ctx->d_wtiles, ctx->tiles_cap));
        CU(dalloc(&ctx->d_sched, (size_t)ctx->tiles_cap * kTileRows));
        CU(dalloc(&ctx->d_wtopo, NP));
        CU(dalloc(&ctx->d_tile_counter, 1));
        CU(dalloc(&ctx->d_tile_ticket, 1)); CU(cudaMemset(ctx->d_tile_ticket, 0, 4));
        r.wtopo = ctx->d_wtopo;
        // worst case tables: every view with three (kMaxClusters+1)-entry plane tables + kMaxClusters thresholds, and the views'
        // RenderLayers blocks 1..3 (FrameConsts::view_ext_off)
        ctx->blob_cap = sizeof(FrameConsts) + V * (3 * (size_t)(kMaxClusters + 1) * 16 + (size_t)kMaxClusters * 4) +
                        sizeof(uint64_t) * 3 * kMaxCameras;
        CU(dalloc(&ctx->d_blob2[0], ctx->blob_cap)); CU(dalloc(&ctx->d_blob2[1], ctx->blob_cap)); CU(dalloc(&ctx->d_blob2[2], ctx->blob_cap));
        ctx->d_blob = ctx->d_blob2[0];
        ctx->d_consts = reinterpret_cast<FrameConsts *>(ctx->d_blob);
        {   // the tail kernels are small and latency-bound: give their CTAs priority over the bulk tile pass
            int lo = 0, hi = 0;
            CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
            CU(cudaStreamCreateWithPriority(&ctx->side_stream, cudaStreamNonBlocking, hi));
            CU(cudaStreamCreateWithPriority(&ctx->clus_stream, cudaStreamNonBlocking, hi));
            CU(cudaEventCreateWithFlags(&ctx->ev_clus, cudaEventDisableTiming));
        }
        CU(cudaEventCreateWithFlags(&ctx->ev_tile, cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&ctx->ev_pub, cudaEventDisableTiming));
        for (cudaEvent_t &e : ctx->ev_side) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        for (cudaEvent_t &e : ctx->ev_expand) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        { const char *e = getenv("B200VIS_PIPELINE"); if (e && e[0] == '0') ctx->pipeline = false; }
        { const char *e = getenv("B200VIS_GT_STAGE"); ctx->gt_stage_full = e && e[0] == 'f'; }
        for (int i = 0; i < b200vis_ctx::kRing; ++i) {
            CU(cudaMallocHost(&ctx->h_ring[i], ctx->blob_cap));
            CU(cudaEventCreateWithFlags(&ctx->ring_ev[i], cudaEventDisableTiming));
        }
        // visible set buffers
        VisibleBufs &vb = ctx->vis;
        vb.words_stride = (uint32_t)((N + 31) / 32 + 2);
        vb.chunks_stride = (vb.words_stride + kChunkWords - 1) / kChunkWords + 1;
        vb.list_stride = (uint32_t)std::max<size_t>(N, 1);
        CU(dalloc(&vb.mask, (size_t)2 * vb.words_stride * V));
        CU(dalloc(&vb.chunk_count, (size_t)3 * kMaxCameras * vb.chunks_stride));
        CU(dalloc(&vb.lists, (size_t)vb.list_stride * V));
        CU(dalloc(&vb.classes, (size_t)vb.list_stride * V));
        CU(dalloc(&ctx->d_cls, NP));
        vb.cls = ctx->d_cls;
        CU(dalloc(&ctx->d_stats, 1));
        CU(cudaMallocHost(&ctx->h_stats, sizeof(DevStats)));
        // lights + clusters
        const size_t Lm = std::max<uint32_t>(cfg->max_lights, 1);
        CU(dalloc(&ctx->d_tag_flag, 1));
        CU(dalloc(&ctx->d_light_ord, N));
        CU(cudaMemset(ctx->d_light_ord, 0xFF, std::max<size_t>(N, 1) * 4));
        CU(dalloc(&ctx->d_light_row, Lm)); CU(dalloc(&ctx->d_light_range, Lm)); CU(dalloc(&ctx->d_light_layers, Lm));
        ClusterBufs &cl = ctx->cl;
        cl.words = (uint32_t)((Lm + 31) / 32); cl.max_lights = cl.words * 32; cl.world = ctx->cfg.world_size;
        cl.rank = cfg->rank; cl.max_views = (uint32_t)V; cl.index_cap = ctx->cfg.max_cluster_indices;
        ctx->lrec_bytes = (size_t)cl.max_lights * 28;
        CU(cudaMalloc(&ctx->d_lrec, 3 * ctx->lrec_bytes)); CU(cudaMemset(ctx->d_lrec, 0, 3 * ctx->lrec_bytes));
        if (cl.world > 1) { CU(cudaMalloc(&ctx->d_lrec_all, cl.world * ctx->lrec_bytes)); CU(cudaMemset(ctx->d_lrec_all, 0, cl.world * ctx->lrec_bytes)); }
        cl.trailer = (uint32_t)std::max<size_t>(V, kMaxViews);
        cl.slab_words = (uint32_t)(V * cl.words * kMaxClusters + cl.trailer);   // bit matrix + per-view farthest_z trailer
        ctx->slab_bytes = (size_t)cl.slab_words * sizeof(uint32_t);
        CU(dalloc(&ctx->d_slab, ctx->slab_bytes / 4));
        cl.send = ctx->d_slab; cl.recv = ctx->d_slab;
        cl.blob = reinterpret_cast<const float *>(ctx->d_blob);   // re-pointed per frame
        CU(dalloc(&cl.offsets, V * (kMaxClusters + 1)));
        CU(dalloc(&cl.indices, V * (size_t)cl.index_cap));
        ctx->stage_bytes = std::max<size_t>(N, 1) * 64;
        CU(cudaMalloc(&ctx->d_stage, ctx->stage_bytes));
        CU(cudaMallocHost(&ctx->h_stage, ctx->stage_bytes));
        return B200VIS_OK;
    }();
    if (rc != B200VIS_OK) { g_create_error = ctx->err; b200vis_destroy(ctx); return rc; }
    *out = ctx;
    return B200VIS_OK;
}

#define CHECK_CTX()                                                        \
    if (!ctx) return B200VIS_ERR_INVALID_ARG;                              \
    CU(cudaSetDevice(ctx->device))

static int32_t join_side(b200vis_ctx *ctx);
static int32_t join_all(b200vis_ctx *ctx);
#define CHECK_CTX_JOIN()                                                   \
    CHECK_CTX();                                                           \
    { const int32_t jrc_ = join_all(ctx); if (jrc_) return jrc_; }

static int32_t check_range(b200vis_ctx *ctx, uint32_t first, uint32_t count, const char *what) {
    if ((uint64_t)first + count > ctx->cfg.max_entities)
        return fail(ctx, B200VIS_ERR_CAPACITY, "%s: rows [%u, %u) exceed max_entities %u", what, first, first + count,
                    ctx->cfg.max_entities);
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_stream(b200vis_ctx *ctx, void *cuda_stream) {
    CHECK_CTX_JOIN();
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_synchronize(b200vis_ctx *ctx) {
    CHECK_CTX_JOIN();
    CU(cudaStreamSynchronize(ctx->stream));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_static_transform_optimizations(b200vis_ctx *ctx, int32_t enabled) {
    if (!ctx) return B200VIS_ERR_INVALID_ARG;
    ctx->static_opt = enabled ? 1 : 0;
    return B200VIS_OK;
}

// ------------------------------------------------------------------------------------------
// execution plan
// ------------------------------------------------------------------------------------------
// Validates the hierarchy (range, cycles), cuts the rows into tiles of <= kTileRows rows --
// preferring cuts at tree boundaries so parents sit in the same tile as their children -- and
// orders the tiles into passes so that a tile's out-of-tile parents are finished by an earlier
// launch.  Forests of small trees need one pass; a tree larger than a tile needs a few.
struct Plan {
    std::vector<uint32_t> topo;          // per row, CTA-per-tile kernels (device_types.cuh T_*)
    std::vector<uint32_t> wtopo;         // per row, k_tile_warp
    std::vector<Tile> tiles;             // sorted by pass
    std::vector<WarpTile> wtiles;        // the same tiles, same order, as warp work items
    std::vector<uint8_t> sched;          // kTileRows bytes per tile: schedule slot -> local row, 0xFF = padding
    std::vector<uint32_t> pass_begin;    // tile index ranges per pass: [pass_begin[p], pass_begin[p+1])
    std::vector<uint32_t> pass_small;
    uint32_t n_ext = 0;                  // rows whose parent sits in another tile
    // The same tiles in creation (= row) order, with what b200vis_edit_topology needs to re-plan some of them: the tile of
    // every row, each tile's pass and the tiles of its out-of-tile parents, and the live children of every row.
    // WarpTile::sched is the creation index, in both orders.
    std::vector<Tile> tiles_c;
    std::vector<WarpTile> wtiles_c;
    std::vector<uint32_t> tile_of, level, n_children;
    std::vector<std::vector<uint32_t>> ext;
    uint32_t cap = kTileRows;            // tile size the rows were cut with
    // edit state (b200vis_edit_topology): the parent array, which rows are alive
    std::vector<uint32_t> parent;
    std::vector<uint8_t> alive;
    uint32_t n = 0, n_dead = 0;
};

static bool split_deep_tiles() {
    static int split_env = -1;
    if (split_env < 0) { const char *e = getenv("B200VIS_SPLIT_DEEP_TILES"); split_env = (e && atoi(e)) ? 1 : 0; }
    return split_env == 1;
}

// Greedy tiling of rows [start, n), cutting at the latest tree boundary inside a full tile; appends to `tiles`.
static void cut_tiles(uint32_t n, const uint32_t *parent, uint32_t start, uint32_t cap, std::vector<Tile> &tiles) {
    const bool split_deep = split_deep_tiles();
    std::vector<uint8_t> marked(n - start, 0);
    while (start < n) {
        uint32_t end = std::min<uint32_t>(n, start + cap);
        if (end < n && parent[end] < n) {          // the cut would split a tree: back up to a boundary
            uint32_t c = end;
            while (c > start + 1 && parent[c] < n) --c;   // c = latest row in (start, end] that starts a tree
            if (c > start && !(parent[c] < n)) end = c;
        }
        {   // k_tile_warp keeps the GlobalTransforms of the rows WITH in-tile children in kWarpParentSlots shared-memory
            // slots: cut the tile before the child that would need one more (only chains and unary-heavy trees get there)
            const uint32_t s0 = (uint32_t)(n - marked.size());
            uint32_t parents = 0;
            for (uint32_t c = start; c < end; ++c) {
                const uint32_t p = parent[c];
                if (p < n && p >= start && !marked[p - s0]) {
                    if (parents == (uint32_t)kWarpParentSlots) { end = c; break; }
                    marked[p - s0] = 1; ++parents;
                }
            }
        }
        // EXPERIMENT (B200VIS_SPLIT_DEEP_TILES=1, off by default): the hierarchy walk of a tile is a serial chain of its
        // levels (DESIGN.md section 7: ~680 cycles per level).  When the first <= 32 rows of a deep tile are exactly its top
        // K levels (level-ordered rows, e.g. one tree in BFS order), cut there: the top becomes a tile of its own, one pass
        // earlier (run by 32-thread CTAs), and the bottom keeps only n_levels - K levels with external parents.
        uint32_t cut = 0;
        if (split_deep && end - start > 64) {
            std::vector<uint32_t> dep(end - start, 0), cnt;
            for (uint32_t r = start; r < end; ++r) {
                const uint32_t p = parent[r];
                dep[r - start] = (p < n && p >= start) ? dep[p - start] + 1 : 0;
                if (dep[r - start] >= cnt.size()) cnt.resize(dep[r - start] + 1, 0);
                cnt[dep[r - start]]++;
            }
            const uint32_t levels = (uint32_t)cnt.size();
            if (levels >= 6) {
                uint32_t rows_above = 0;
                for (uint32_t K = 1; K + 2 <= levels; ++K) {       // rows with depth < K
                    rows_above += cnt[K - 1];
                    if (rows_above > 32) break;
                    bool prefix = true;                              // they must be exactly the first rows_above rows
                    for (uint32_t i = 0; i < end - start && prefix; ++i) prefix = (dep[i] < K) == (i < rows_above);
                    if (prefix && K >= 2) cut = rows_above;
                }
            }
        }
        for (uint32_t part = 0; part < (cut ? 2u : 1u); ++part) {
            const uint32_t b = (part == 0) ? start : start + cut, e = (cut && part == 0) ? start + cut : end;
            Tile t; t.base = b; t.n_rows = (uint16_t)(e - b); t.n_levels = 1; t.warp_sync_mask = 0xFFFFFFFFu; t.top_levels = 0; t.lvl_warps = 0;
            tiles.push_back(t);
        }
        start = end;
    }
}

// Plans one tile (t.base, t.n_rows set): the topo / wtopo words of its rows, its level data, schedule and warp work item,
// and the tiles of its out-of-tile parents (sorted, unique).  T_HAS_CHILDREN is "has a child anywhere" (n_children[r] > 0);
// tile_of(p) gives the tile of a row before t.base.  Returns the rows with an out-of-tile parent, or -1 when the rows with
// in-tile children exceed the warp kernel's kWarpParentSlots (only an edit can produce such a tile: the tiler cuts before).
template <class TileOf>
static int64_t plan_tile(const uint32_t *parent, const uint32_t *n_children, TileOf tile_of, Tile &t, WarpTile &w,
                         uint32_t creation_index, uint8_t *sch, uint32_t *topo, uint32_t *wtopo, std::vector<uint32_t> &ext) {
    const uint32_t b = t.base, nr = t.n_rows;
    t.n_levels = 1; t.warp_sync_mask = 0xFFFFFFFFu; t.top_levels = 0; t.lvl_warps = 0;
    uint32_t ldepth[kTileRows];
    uint8_t local_kids[kTileRows] = {};   // rows with children IN THEIR OWN TILE (a child in a later tile reads its parent from HBM)
    ext.clear();
    int64_t n_ext = 0;
    // topo words, in-tile depth, tile levels
    for (uint32_t i = 0; i < nr; ++i) {
        const uint32_t r = b + i, p = parent[r];
        uint32_t wd = 0;
        ldepth[i] = 0;
        if (p == kNoParent) wd |= T_ROOT;
        else if (p == kDetached) wd |= T_DETACHED;
        else if (p >= b) {
            ldepth[i] = ldepth[p - b] + 1;
            local_kids[p - b] = 1;
            wd |= (p - b) | (ldepth[i] << 9);
            t.n_levels = std::max<uint16_t>(t.n_levels, (uint16_t)(ldepth[i] + 1));
            // a level keeps its warp-sync bit only while every parent->child edge into it stays inside one warp
            if (ldepth[i] < 32 && ((p - b) >> 5) != (i >> 5)) t.warp_sync_mask &= ~(1u << ldepth[i]);
        } else {
            wd |= T_EXT_PARENT;
            ++n_ext;
            ext.push_back(tile_of(p));
        }
        if (n_children[r]) wd |= T_HAS_CHILDREN;
        topo[i] = wd;
    }
    std::sort(ext.begin(), ext.end());
    ext.erase(std::unique(ext.begin(), ext.end()), ext.end());
    {   // top_levels: the leading depth levels whose rows all sit among the tile's first 32 rows
        uint32_t max_local[kTileRows] = {};
        for (uint32_t i = 0; i < nr; ++i) max_local[ldepth[i]] = std::max(max_local[ldepth[i]], i);
        uint32_t K = 0;
        while (K < t.n_levels && max_local[K] < 32u) ++K;
        static int cap_env = -1;      // B200VIS_TOP_LEVELS_CAP: how many levels the scout may take (experiment knob)
        if (cap_env < 0) { const char *e = getenv("B200VIS_TOP_LEVELS_CAP"); cap_env = e ? atoi(e) : 255; }
        if (K > (uint32_t)cap_env) K = (uint32_t)cap_env;
        t.top_levels = (t.n_levels > 1) ? K : 0u;       // flat tiles have nothing to walk ahead
    }
    {   // lvl_warps: which warps meet at which level hand-over (named barriers, k_propagate_cull_tma)
        static int level_sync = -1;     // B200VIS_LEVEL_SYNC=cta: keep the CTA-wide level barriers (A/B switch)
        if (level_sync < 0) { const char *e = getenv("B200VIS_LEVEL_SYNC"); level_sync = (e && e[0] == 'c') ? 0 : 1; }
        if (level_sync && t.n_levels >= 2 && t.n_levels <= 8) {      // seven barrier ids per tile parity (levels 1..7)
            uint32_t lv[kTileRows / 32] = {};          // per warp: bit l = the warp holds a row of in-tile depth l (a detached
            for (uint32_t i = 0; i < nr; ++i)          // row has depth 0: it publishes "not visited" to its children)
                lv[i >> 5] |= 1u << ldepth[i];
            unsigned long long packed = 0;
            for (uint32_t l = 1; l < t.n_levels; ++l) {
                unsigned long long c = 0;
                for (uint32_t wi = 0; wi < (uint32_t)kTileRows / 32u; ++wi) c += ((lv[wi] >> (l - 1)) & 3u) ? 1u : 0u;
                packed |= c << (4u * l);
            }
            t.lvl_warps = packed;
        }
    }
    // ---- warp work item: schedule, parent slots, wtopo -------------------------------------------------------------
    // rows in (depth, row) order: counting sort by in-tile depth
    uint32_t level_count[kTileRows + 1] = {}, order[kTileRows], slot_of[kTileRows] = {};
    for (uint32_t i = 0; i < nr; ++i) level_count[ldepth[i] + 1]++;
    for (uint32_t l = 0; l < t.n_levels; ++l) level_count[l + 1] += level_count[l];
    { uint32_t cur[kTileRows];
      for (uint32_t l = 0; l < t.n_levels; ++l) cur[l] = level_count[l];
      for (uint32_t i = 0; i < nr; ++i) order[cur[ldepth[i]]++] = i; }
    // slots: a level with >= 32 rows starts on a chunk boundary when the padding still fits into kTileRows slots
    memset(sch, 0xFF, kTileRows);
    uint32_t pos = 0, next_slot = 0;
    for (uint32_t l = 0; l < t.n_levels; ++l) {
        const uint32_t lb = level_count[l], le = level_count[l + 1], cnt = le - lb;
        if ((pos & 31u) && cnt >= 32u) {
            const uint32_t padded = (pos + 31u) & ~31u;
            if (padded + (nr - lb) <= (uint32_t)kTileRows) pos = padded;
        }
        for (uint32_t i = lb; i < le; ++i) {
            sch[pos++] = (uint8_t)order[i];
            if (local_kids[order[i]]) slot_of[order[i]] = next_slot++;
        }
    }
    if (next_slot > (uint32_t)kWarpParentSlots) return -1;
    memset(&w, 0, sizeof w);
    w.base = b; w.n_rows = (uint16_t)nr; w.n_chunks = (uint8_t)((pos + 31u) / 32u); w.sched = creation_index;
    for (uint32_t c = 0; c < w.n_chunks; ++c) {
        bool contig = true; int64_t delta = 0; bool have = false;
        for (uint32_t lane = 0; lane < 32; ++lane) {
            const uint8_t lr = sch[c * 32 + lane];
            if (lr == 0xFF && nr != (uint32_t)kTileRows) continue;   // padding (a full tile has none: 0xFF is row 255)
            const int64_t d = (int64_t)lr - (int64_t)lane;
            if (!have) { delta = d; have = true; } else if (d != delta) contig = false;
            if (ldepth[lr] > 0) w.nonroot[c] |= 1u << lane;
        }
        if (contig) w.contig |= (uint8_t)(1u << c);
    }
    for (uint32_t i = 0; i < nr; ++i) {
        uint32_t wd = topo[i] & 0xF0000000u;      // T_HAS_CHILDREN stays the reference's "has a Children component"
        if (local_kids[i]) wd |= W_HAS_SLOT | (slot_of[i] << 8);
        wd |= ldepth[i] & 0xFFu;
        if (ldepth[i]) wd |= slot_of[parent[b + i] - b] << 15;
        wtopo[i] = wd;
    }
    return n_ext;
}

// Passes from the tile graph (a tile runs one pass after the latest of its out-of-tile parents' tiles), then the tiles
// sorted by pass.  O(tiles + external edges): a parent row precedes its children, so ext tiles have smaller indices.
static void order_passes(Plan &plan) {
    const size_t T = plan.tiles_c.size();
    plan.level.assign(T, 0);
    for (size_t ti = 0; ti < T; ++ti)
        for (uint32_t e : plan.ext[ti]) plan.level[ti] = std::max(plan.level[ti], plan.level[e] + 1);
    const uint32_t n_pass = T ? *std::max_element(plan.level.begin(), plan.level.end()) + 1 : 0;
    plan.pass_begin.assign(n_pass + 1, 0);
    for (uint32_t lv : plan.level) plan.pass_begin[lv + 1]++;
    for (uint32_t p = 0; p < n_pass; ++p) plan.pass_begin[p + 1] += plan.pass_begin[p];
    plan.tiles.resize(T);
    plan.wtiles.resize(T);
    std::vector<uint32_t> cursor(plan.pass_begin.begin(), plan.pass_begin.end() - (n_pass ? 1 : 0));
    plan.pass_small.assign(n_pass, 0);
    // within a pass: the small tiles (<= 32 rows, only produced by B200VIS_SPLIT_DEEP_TILES) first, then the rest
    const bool split_deep = split_deep_tiles();
    for (int small = 1; small >= 0; --small)
        for (size_t i = 0; i < T; ++i) {
            const bool is_small = split_deep && plan.tiles_c[i].n_rows <= 32;
            if ((int)is_small != small) continue;
            const uint32_t at = cursor[plan.level[i]]++;
            plan.tiles[at] = plan.tiles_c[i];
            plan.wtiles[at] = plan.wtiles_c[i];       // .sched keeps pointing at the tile's block in creation order
            if (is_small) plan.pass_small[plan.level[i]]++;
        }
}

// Validates the hierarchy (range, cycles), cuts the rows into tiles of <= kTileRows rows --
// preferring cuts at tree boundaries so parents sit in the same tile as their children -- and
// orders the tiles into passes so that a tile's out-of-tile parents are finished by an earlier
// launch.  Forests of small trees need one pass; a tree larger than a tile needs a few.
static int32_t build_plan(b200vis_ctx *ctx, uint32_t n, const uint32_t *parent, uint32_t cap, Plan &plan) {
    if (cap < 32) cap = 32;
    if (cap > (uint32_t)kTileRows) cap = kTileRows;
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t p = parent[r];
        if (p == kNoParent || p == kDetached) continue;
        if (p >= n) return fail(ctx, B200VIS_ERR_PARENT_OUT_OF_RANGE, "row %u: parent %u out of range (n=%u)", r, p, n);
    }
    {   // cycle check: every chain must end at a root / detached row
        std::vector<uint8_t> color(n, 0);
        std::vector<uint32_t> path;
        for (uint32_t r = 0; r < n; ++r) {
            if (color[r]) continue;
            path.clear();
            uint32_t c = r;
            while (true) {
                if (color[c] == 2) break;
                if (color[c] == 1) return fail(ctx, B200VIS_ERR_HIERARCHY_CYCLE, "hierarchy cycle through row %u", c);
                color[c] = 1; path.push_back(c);
                const uint32_t p = parent[c];
                if (p >= n) break;
                c = p;
            }
            for (uint32_t x : path) color[x] = 2;
        }
    }
    for (uint32_t r = 0; r < n; ++r)
        if (parent[r] < n && parent[r] >= r)
            return fail(ctx, B200VIS_ERR_UNSUPPORTED,
                        "row %u has parent %u >= itself: rows must be in topological order (use b200vis_plan_row_order)", r,
                        parent[r]);
    plan.cap = cap; plan.n = n; plan.n_dead = 0;
    plan.tiles_c.clear();
    cut_tiles(n, parent, 0, cap, plan.tiles_c);
    const size_t T = plan.tiles_c.size();
    plan.tile_of.resize(n);
    for (size_t ti = 0; ti < T; ++ti)
        for (uint32_t r = plan.tiles_c[ti].base; r < plan.tiles_c[ti].base + plan.tiles_c[ti].n_rows; ++r) plan.tile_of[r] = (uint32_t)ti;
    plan.n_children.assign(n, 0);
    for (uint32_t r = 0; r < n; ++r) if (parent[r] < n) plan.n_children[parent[r]]++;
    plan.topo.resize(n); plan.wtopo.resize(n);
    plan.wtiles_c.resize(T);
    plan.sched.assign(T * (size_t)kTileRows, 0xFF);
    plan.ext.assign(T, {});
    plan.n_ext = 0;
    const uint32_t *tile_of = plan.tile_of.data();
    for (size_t ti = 0; ti < T; ++ti) {
        const uint32_t b = plan.tiles_c[ti].base;
        plan.n_ext += (uint32_t)plan_tile(parent, plan.n_children.data(), [tile_of](uint32_t p) { return tile_of[p]; }, plan.tiles_c[ti],
                                          plan.wtiles_c[ti], (uint32_t)ti, plan.sched.data() + ti * (size_t)kTileRows,
                                          plan.topo.data() + b, plan.wtopo.data() + b, plan.ext[ti]);
    }
    order_passes(plan);
    return B200VIS_OK;
}

// ---- incremental re-planning (b200vis_edit_topology) ----------------------------------------------------------------
struct TopologyEdit {
    uint32_t n_despawn; const uint32_t *despawn;
    uint32_t n_reparent; const uint32_t *reparent; const uint32_t *new_parent;
    uint32_t n_spawn; const uint32_t *spawn_parent;
};
struct EditResult {
    std::vector<uint32_t> tiles;                           // re-planned tiles (creation index), ascending
    std::vector<std::pair<uint32_t, uint32_t>> ranges;     // their row ranges [first, end), ascending and disjoint
    uint32_t rows = 0;                                     // rows re-planned
};

// Applies one frame's despawns, reparents and spawns to the plan, re-planning only the tiles they touch: the tiles
// holding a despawned or reparented row, the tiles of parents that gain their first or lose their last child, and for
// spawns the last tile (if not full) together with the appended rows, cut by the same greedy tiler.  Host work is
// O(edited rows + re-planned tiles x kTileRows + tiles).  All or nothing: on error `hp` is unchanged.
static int32_t edit_plan(b200vis_ctx *ctx, Plan &hp, uint32_t max_rows, const TopologyEdit &ed, EditResult &res) {
    const uint32_t n = hp.n, n2 = n + ed.n_spawn;
    if ((uint64_t)n + ed.n_spawn > max_rows)
        return fail(ctx, B200VIS_ERR_CAPACITY, "edit_topology: %u + %u rows exceed max_entities %u", n, ed.n_spawn, max_rows);
    if (split_deep_tiles()) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "edit_topology: not with B200VIS_SPLIT_DEEP_TILES");
    // ---- validation (nothing is touched) ----
    std::vector<uint32_t> ds(ed.despawn, ed.despawn + ed.n_despawn);
    std::sort(ds.begin(), ds.end());
    auto despawned = [&](uint32_t r) { return std::binary_search(ds.begin(), ds.end(), r); };
    for (size_t i = 0; i < ds.size(); ++i) {
        if (ds[i] >= n || !hp.alive[ds[i]]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: despawned row %u is out of range or dead", ds[i]);
        if (i && ds[i] == ds[i - 1]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: row %u is despawned twice", ds[i]);
    }
    {   // despawn is recursive: every live child of a despawned row is despawned in the same call
        std::vector<uint32_t> kids(ds.size(), 0);
        for (uint32_t d : ds) {
            const uint32_t p = hp.parent[d];
            if (p < n && despawned(p)) kids[std::lower_bound(ds.begin(), ds.end(), p) - ds.begin()]++;
        }
        for (size_t i = 0; i < ds.size(); ++i)
            if (kids[i] != hp.n_children[ds[i]])
                return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: despawned row %u keeps %u live children (despawn them too, or reparent them first)",
                            ds[i], hp.n_children[ds[i]] - kids[i]);
    }
    {
        std::vector<uint32_t> rp(ed.reparent, ed.reparent + ed.n_reparent);
        std::sort(rp.begin(), rp.end());
        for (size_t i = 1; i < rp.size(); ++i)
            if (rp[i] == rp[i - 1]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: row %u is reparented twice", rp[i]);
    }
    for (uint32_t j = 0; j < ed.n_reparent; ++j) {
        const uint32_t r = ed.reparent[j], p = ed.new_parent[j];
        if (r >= n || !hp.alive[r] || despawned(r)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: reparented row %u is out of range or dead", r);
        if (p == kNoParent || p == kDetached) continue;
        if (p >= n) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: new parent %u of row %u is out of range", p, r);
        if (p >= r) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "edit_topology: new parent %u of row %u breaks the row order (compact with set_topology)", p, r);
        if (!hp.alive[p] || despawned(p)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: new parent %u of row %u is dead", p, r);
    }
    for (uint32_t k = 0; k < ed.n_spawn; ++k) {
        const uint32_t r = n + k, p = ed.spawn_parent[k];
        if (p == kNoParent || p == kDetached) continue;
        if (p >= n2) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: parent %u of spawned row %u is out of range", p, r);
        if (p >= r) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "edit_topology: parent %u of spawned row %u is a later row of the batch", p, r);
        if (p < n && (!hp.alive[p] || despawned(p))) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: parent %u of spawned row %u is dead", p, r);
    }
    // ---- apply to the hierarchy (undone if a re-planned tile turns out unplannable) ----
    std::vector<std::pair<uint32_t, uint32_t>> old_parent;          // (row, parent before the edit)
    std::vector<uint32_t> dirty;
    auto touch_parent = [&](uint32_t p, int delta) {                 // a parent gains / loses a child
        if (p >= n2) return;
        const uint32_t before = hp.n_children[p];
        hp.n_children[p] = before + delta;
        if (p < n && ((before == 0) != (hp.n_children[p] == 0))) dirty.push_back(hp.tile_of[p]);   // T_HAS_CHILDREN flips
    };
    hp.parent.resize(n2); hp.alive.resize(n2, 1); hp.n_children.resize(n2, 0);
    for (uint32_t d : ds) {
        old_parent.emplace_back(d, hp.parent[d]);
        touch_parent(hp.parent[d], -1);
        hp.parent[d] = kDetached; hp.alive[d] = 0;
        dirty.push_back(hp.tile_of[d]);
    }
    for (uint32_t j = 0; j < ed.n_reparent; ++j) {
        const uint32_t r = ed.reparent[j];
        old_parent.emplace_back(r, hp.parent[r]);
        touch_parent(hp.parent[r], -1);
        hp.parent[r] = ed.new_parent[j];
        touch_parent(hp.parent[r], +1);
        dirty.push_back(hp.tile_of[r]);
    }
    for (uint32_t k = 0; k < ed.n_spawn; ++k) {
        hp.parent[n + k] = ed.spawn_parent[k];
        touch_parent(ed.spawn_parent[k], +1);
    }
    auto undo = [&]() {
        for (size_t i = old_parent.size(); i-- > 0;) {
            const uint32_t r = old_parent[i].first;
            touch_parent(hp.parent[r], -1);
            hp.parent[r] = old_parent[i].second;
            touch_parent(hp.parent[r], +1);
            hp.alive[r] = 1;
        }
        for (uint32_t k = 0; k < ed.n_spawn; ++k) touch_parent(ed.spawn_parent[k], -1);
        hp.parent.resize(n); hp.alive.resize(n); hp.n_children.resize(n);
    };
    // ---- re-plan ----
    const uint32_t T = (uint32_t)hp.tiles_c.size();
    uint32_t sfx_tile = T, s = n;            // spawns: tiles [sfx_tile, ...) are cut again from row s
    if (ed.n_spawn && T && hp.tiles_c[T - 1].n_rows < hp.cap) { sfx_tile = T - 1; s = hp.tiles_c[T - 1].base; }
    std::sort(dirty.begin(), dirty.end());
    dirty.erase(std::unique(dirty.begin(), dirty.end()), dirty.end());
    while (!dirty.empty() && dirty.back() >= sfx_tile) dirty.pop_back();
    std::vector<Tile> sfx;
    if (ed.n_spawn) cut_tiles(n2, hp.parent.data(), s, hp.cap, sfx);
    std::vector<uint32_t> sfx_tile_of(n2 - s);
    for (size_t i = 0; i < sfx.size(); ++i)
        for (uint32_t r = sfx[i].base; r < sfx[i].base + sfx[i].n_rows; ++r) sfx_tile_of[r - s] = sfx_tile + (uint32_t)i;
    const uint32_t *tile_of = hp.tile_of.data(), *sto = sfx_tile_of.data();
    auto tile_of_row = [tile_of, sto, s](uint32_t p) { return p >= s ? sto[p - s] : tile_of[p]; };
    const size_t n_new = dirty.size() + sfx.size();
    std::vector<Tile> nt(n_new);
    std::vector<WarpTile> nw(n_new);
    std::vector<std::vector<uint32_t>> next(n_new);
    std::vector<uint8_t> nsched(n_new * (size_t)kTileRows);
    std::vector<uint32_t> ntopo, nwtopo;
    uint32_t rows = 0;
    for (size_t i = 0; i < n_new; ++i) rows += i < dirty.size() ? hp.tiles_c[dirty[i]].n_rows : sfx[i - dirty.size()].n_rows;
    ntopo.resize(rows); nwtopo.resize(rows);
    for (size_t i = 0, at = 0; i < n_new; ++i) {
        const bool d = i < dirty.size();
        nt[i] = d ? hp.tiles_c[dirty[i]] : sfx[i - dirty.size()];
        const uint32_t ci = d ? dirty[i] : sfx_tile + (uint32_t)(i - dirty.size());
        if (plan_tile(hp.parent.data(), hp.n_children.data(), tile_of_row, nt[i], nw[i], ci, nsched.data() + i * (size_t)kTileRows,
                      ntopo.data() + at, nwtopo.data() + at, next[i]) < 0) {
            undo();
            return fail(ctx, B200VIS_ERR_UNSUPPORTED, "edit_topology: tile at row %u would need more than %d parent slots (compact with set_topology)",
                        nt[i].base, kWarpParentSlots);
        }
        at += nt[i].n_rows;
    }
    // ---- commit ----
    hp.tiles_c.resize(sfx_tile + sfx.size()); hp.wtiles_c.resize(sfx_tile + sfx.size()); hp.ext.resize(sfx_tile + sfx.size());
    hp.sched.resize(hp.tiles_c.size() * (size_t)kTileRows);
    hp.topo.resize(n2); hp.wtopo.resize(n2); hp.tile_of.resize(n2);
    for (uint32_t r = s; r < n2; ++r) hp.tile_of[r] = sfx_tile_of[r - s];
    res.tiles.clear(); res.ranges.clear(); res.rows = rows;
    for (size_t i = 0, at = 0; i < n_new; ++i) {
        const uint32_t ci = i < dirty.size() ? dirty[i] : sfx_tile + (uint32_t)(i - dirty.size());
        hp.tiles_c[ci] = nt[i]; hp.wtiles_c[ci] = nw[i]; hp.ext[ci].swap(next[i]);
        memcpy(hp.sched.data() + (size_t)ci * kTileRows, nsched.data() + i * (size_t)kTileRows, kTileRows);
        memcpy(hp.topo.data() + nt[i].base, ntopo.data() + at, nt[i].n_rows * 4u);
        memcpy(hp.wtopo.data() + nt[i].base, nwtopo.data() + at, nt[i].n_rows * 4u);
        at += nt[i].n_rows;
        res.tiles.push_back(ci);
        if (!res.ranges.empty() && res.ranges.back().second == nt[i].base) res.ranges.back().second += nt[i].n_rows;
        else res.ranges.emplace_back(nt[i].base, nt[i].base + nt[i].n_rows);
    }
    hp.n = n2; hp.n_dead += (uint32_t)ds.size();
    hp.n_ext = 0;     // not tracked across edits (only set_topology's choice of tile size reads it)
    order_passes(hp);
    return B200VIS_OK;
}

static int32_t plan_world(b200vis_ctx *ctx, uint32_t n, const uint32_t *parent, Plan &plan);

// The host half of b200vis_compact_topology: the survivors (live rows, and the dead rows in `held` that results still
// name), the reparents applied, the survivors renumbered in b200vis_plan_row_order's order of their current order, and
// the plan set_topology builds for the new parent array (cap == 0: with its tile-size search).  Writes the new plan to
// `out`; `hp` is only read.
static int32_t compact_plan(b200vis_ctx *ctx, const Plan &hp, uint32_t n_reparent, const uint32_t *reparent, const uint32_t *new_parent,
                            const std::vector<uint32_t> &held, uint32_t cap, Plan &out, std::vector<uint32_t> &old_to_new,
                            std::vector<uint32_t> &new_to_old) {
    const uint32_t n = hp.n;
    std::vector<uint32_t> par(hp.parent);
    std::vector<uint8_t> keep(hp.alive);
    for (uint32_t r : held) {
        if (r >= n || hp.alive[r]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "compact_topology: held row %u is out of range or live", r);
        keep[r] = 1;
    }
    {
        std::vector<uint32_t> rp(reparent, reparent + n_reparent);
        std::sort(rp.begin(), rp.end());
        for (size_t i = 1; i < rp.size(); ++i)
            if (rp[i] == rp[i - 1]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "compact_topology: row %u is reparented twice", rp[i]);
    }
    for (uint32_t j = 0; j < n_reparent; ++j) {
        const uint32_t r = reparent[j], p = new_parent[j];
        if (r >= n || !hp.alive[r]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "compact_topology: reparented row %u is out of range or dead", r);
        if (p != kNoParent && p != kDetached && (p >= n || !hp.alive[p]))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "compact_topology: new parent %u of row %u is out of range or dead", p, r);
        par[r] = p;
    }
    // survivors in their current order; a live row's parent is live (despawns are recursive), a dead row is detached
    std::vector<uint32_t> surv, s_of(n, kNoParent);
    for (uint32_t r = 0; r < n; ++r)
        if (keep[r]) { s_of[r] = (uint32_t)surv.size(); surv.push_back(r); }
    const uint32_t ns = (uint32_t)surv.size();
    std::vector<uint32_t> ps(ns), ord(ns);
    for (uint32_t i = 0; i < ns; ++i) { const uint32_t p = par[surv[i]]; ps[i] = p < n ? s_of[p] : p; }
    if (b200vis_plan_row_order(ns, ps.data(), ord.data()) != B200VIS_OK)
        return fail(ctx, B200VIS_ERR_HIERARCHY_CYCLE, "compact_topology: the reparents make a hierarchy cycle");
    old_to_new.assign(n, kNoParent);
    new_to_old.resize(ns);
    for (uint32_t i = 0; i < ns; ++i) { new_to_old[i] = surv[ord[i]]; old_to_new[new_to_old[i]] = i; }
    std::vector<uint32_t> pn(ns);
    for (uint32_t i = 0; i < ns; ++i) { const uint32_t p = par[new_to_old[i]]; pn[i] = p < n ? old_to_new[p] : p; }
    const int32_t rc = cap ? build_plan(ctx, ns, pn.data(), cap, out) : plan_world(ctx, ns, pn.data(), out);
    if (rc) return rc;
    out.parent = std::move(pn);
    out.alive.resize(ns);
    out.n_dead = 0;
    for (uint32_t i = 0; i < ns; ++i) { out.alive[i] = hp.alive[new_to_old[i]]; out.n_dead += out.alive[i] ? 0u : 1u; }
    return B200VIS_OK;
}

static void free_plan(Plan *p) { delete p; }

// the pass ranges of a plan, and which passes may run the named-barrier schedule
static void install_passes(b200vis_ctx *ctx, const Plan &plan) {
    const std::vector<uint32_t> &pass_begin = plan.pass_begin;
    ctx->pass_begin = pass_begin;
    ctx->pass_small = plan.pass_small;
    ctx->pass_named.assign(pass_begin.empty() ? 0 : pass_begin.size() - 1, 1);
    for (size_t pi = 0; pi + 1 < pass_begin.size(); ++pi)
        for (uint32_t ti = pass_begin[pi]; ti < pass_begin[pi + 1]; ++ti)
            if (plan.tiles[ti].n_levels > 1 && plan.tiles[ti].lvl_warps == 0ull) { ctx->pass_named[pi] = 0; break; }
}

// The plan of a whole world, as set_topology and the compaction install it.  Tile size: a tile is one WARP's work item, and
// the machine has ~4700 resident warps: small scenes get smaller tiles (more warps busy) as long as that does not split
// trees across tiles (more passes / parents read from HBM).
static int32_t plan_world(b200vis_ctx *ctx, uint32_t n, const uint32_t *parent, Plan &plan) {
    int32_t rc = build_plan(ctx, n, parent, kTileRows, plan);
    if (rc != B200VIS_OK) return rc;
    static int cap_env = -1;
    if (cap_env < 0) { const char *e = getenv("B200VIS_TILE_ROWS"); cap_env = e ? atoi(e) : 0; }
    uint32_t target = cap_env > 0 ? (uint32_t)cap_env : (uint32_t)std::min<uint64_t>(kTileRows, (((uint64_t)n / 9472u) + 31u) / 32u * 32u);
    if (target < 32) target = 32;
    for (uint32_t cap = target; cap < (uint32_t)kTileRows; cap *= 2) {
        Plan q;
        if (build_plan(ctx, n, parent, cap, q) != B200VIS_OK) break;
        if (q.pass_begin.size() <= plan.pass_begin.size() && q.n_ext <= plan.n_ext) { plan = std::move(q); break; }
    }
    return B200VIS_OK;
}

// the slot -> row maps of b200vis_set_tables follow the row numbering
static int32_t tables_unmap_all(b200vis_ctx *ctx);
static int32_t make_keys_resident(b200vis_ctx *ctx);
static int32_t tables_unmap_rows(b200vis_ctx *ctx, uint32_t n_rows, const uint32_t *rows);
static void tables_renumber(b200vis_ctx *ctx, const std::vector<uint32_t> &old_to_new);
static int32_t flush_table_updates(b200vis_ctx *ctx);

// A new plan (set, edit or compaction of the topology): kernel 1b's staging hints are sized to the tile descriptors and
// start at full staging.  Ordered on `st` behind the plan's upload.
static int32_t reset_tile_hints(b200vis_ctx *ctx, cudaStream_t st) {
    if (ctx->hint_cap < ctx->tiles_cap) {
        CU(cudaStreamSynchronize(st));
        cudaFree(ctx->d_tile_hint);
        ctx->d_tile_hint = nullptr; ctx->hint_cap = 0;
        CU(dalloc(&ctx->d_tile_hint, ctx->tiles_cap));
        ctx->hint_cap = ctx->tiles_cap;
    }
    CU(cudaMemsetAsync(ctx->d_tile_hint, 1, ctx->hint_cap, st));
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_topology(b200vis_ctx *ctx, uint32_t n, const uint32_t *parent, const uint64_t *entity_bits) {
    CHECK_CTX_JOIN();
    if (n && (!parent || !entity_bits)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_topology: null array");
    if (n > ctx->cfg.max_entities) return fail(ctx, B200VIS_ERR_CAPACITY, "set_topology: %u rows > max_entities %u", n, ctx->cfg.max_entities);
    Plan plan;
    int32_t rc = plan_world(ctx, n, parent, plan);
    if (rc != B200VIS_OK) return rc;
    ctx->shadow_emit_ready = false;   // rows and rank order change: the last shadow run's bits name other entities
    std::vector<uint32_t> &topo = plan.topo; std::vector<Tile> &tiles = plan.tiles;
    if (tiles.size() > ctx->tiles_cap) {
        void *old[] = {ctx->d_tiles, ctx->d_wtiles, ctx->d_sched};
        for (void *q : old) if (q) cudaFree(q);
        ctx->d_tiles = nullptr; ctx->d_wtiles = nullptr; ctx->d_sched = nullptr; ctx->tiles_cap = (uint32_t)tiles.size() + 1024;
        CU(dalloc(&ctx->d_tiles, ctx->tiles_cap));
        CU(dalloc(&ctx->d_wtiles, ctx->tiles_cap));
        CU(dalloc(&ctx->d_sched, (size_t)ctx->tiles_cap * kTileRows));
    }
    // Entity::to_bits() order -> rank
    bool sorted = true;
    for (uint32_t r = 1; r < n && sorted; ++r) sorted = entity_bits[r - 1] < entity_bits[r];
    std::vector<uint32_t> order, rank;
    if (!sorted) {
        order.resize(n); std::iota(order.begin(), order.end(), 0u);
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return entity_bits[a] < entity_bits[b]; });
        rank.resize(n);
        for (uint32_t i = 0; i < n; ++i) rank[order[i]] = i;
    }
    cudaStream_t st = ctx->stream;
    if (ctx->gt_ext_pending) {     // a new world: GlobalTransforms written into the old one are no longer pending
        launch_clear_gt_ext(st, ctx->rows, ctx->n);
        CU(cudaGetLastError());
        ctx->gt_ext_pending = false;
    }
    CU(cudaStreamSynchronize(st));   // the vectors below are pageable and short-lived: copy synchronously
    CU(cudaMemcpy(ctx->rows.topo, topo.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ctx->d_parent, parent, (size_t)n * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ctx->d_tiles, tiles.data(), tiles.size() * sizeof(Tile), cudaMemcpyHostToDevice));
    if ((rc = reset_tile_hints(ctx, st))) return rc;
    CU(cudaMemcpy(ctx->d_wtiles, plan.wtiles.data(), plan.wtiles.size() * sizeof(WarpTile), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ctx->d_sched, plan.sched.data(), plan.sched.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ctx->d_wtopo, plan.wtopo.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    if (!sorted) {
        CU(cudaMemcpy(ctx->d_rank, rank.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(ctx->d_row_of_rank, order.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    }
    install_passes(ctx, plan);
    ctx->rank_identity = sorted;
    ctx->n = n;
    ctx->rows.n = n;
    ctx->vis.n_words = (n + 31) / 32;
    ctx->vis.n_chunks = (ctx->vis.n_words + kChunkWords - 1) / kChunkWords;
    // fresh accumulation state
    CU(cudaMemset(ctx->vis.mask, 0, (size_t)2 * ctx->vis.words_stride * ctx->cfg.max_views * 4));
    CU(cudaMemset(ctx->vis.chunk_count, 0, (size_t)3 * kMaxCameras * ctx->vis.chunks_stride * 4));
    CU(cudaMemset(ctx->d_stats, 0, sizeof(DevStats)));
    CU(cudaMemset(ctx->d_slab, 0, ctx->slab_bytes));
    if (ctx->diff.prev) CU(cudaMemset(ctx->diff.prev, 0, (size_t)ctx->vis.words_stride * ctx->cfg.max_views * 4));   // ranks changed: old list = empty
    if (ctx->sdiff.added) {                      // ... and every shadow diff slot: the next run reports every list as added
        CU(cudaMemset(ctx->sdiff.prev, 0, (size_t)ctx->sdiff_max_slots * 6 * ctx->vis.words_stride * 4));
        CU(cudaMemset(ctx->sdiff.prev_count, 0, (size_t)ctx->sdiff_max_slots * 6 * ctx->vis.chunks_stride * 4));
        std::fill(ctx->sdiff_held.begin(), ctx->sdiff_held.end(), 0);
    }
    if (ctx->vdiff.added) {                      // ... and every view diff slot
        CU(cudaMemset(ctx->vdiff.prev, 0, (size_t)ctx->vdiff_max_slots * 8 * ctx->vis.words_stride * 4));
        CU(cudaMemset(ctx->vdiff.prev_count, 0, (size_t)ctx->vdiff_max_slots * ctx->vis.chunks_stride * 4));
        std::fill(ctx->vdiff_held.begin(), ctx->vdiff_held.end(), 0);
    }
    ctx->topology_set = true;
    ctx->gt_aos_valid = false;
    {   // what b200vis_edit_topology starts from: the plan, and the keys in rank order (uploaded by the first merge)
        if (!ctx->hplan) ctx->hplan = new Plan();
        plan.parent.assign(parent, parent + n); plan.alive.assign(n, 1);
        *ctx->hplan = std::move(plan);
        ctx->h_keys.resize(n);
        for (uint32_t i = 0; i < n; ++i) ctx->h_keys[i] = entity_bits[sorted ? i : order[i]];
        ctx->keys_resident = false;
        ctx->max_key = n ? ctx->h_keys[n - 1] : 0;
    }
    if (ctx->ent_sink_d || ctx->shsink.entities || ctx->sdiff.added || ctx->vdiff.added) { const int32_t krc = make_keys_resident(ctx); if (krc) return krc; }   // the Entity sinks read them
    return tables_unmap_all(ctx);
}

// The keys in rank order on the device (uploaded from the host copy if they are not there yet).  Once resident, the edits
// and compactions keep them so.
static int32_t make_keys_resident(b200vis_ctx *ctx) {
    if (ctx->keys_resident) return B200VIS_OK;
    if (!ctx->d_keys) CU(dalloc(&ctx->d_keys, ctx->cfg.max_entities));
    CU(cudaStreamSynchronize(ctx->stream));
    if (!ctx->h_keys.empty()) CU(cudaMemcpy(ctx->d_keys, ctx->h_keys.data(), ctx->h_keys.size() * 8, cudaMemcpyHostToDevice));
    ctx->keys_resident = true;
    std::vector<uint64_t>().swap(ctx->h_keys);
    return B200VIS_OK;
}

static int32_t grow_edit_staging(b200vis_ctx *ctx, size_t bytes) {
    if (bytes <= ctx->h_edit_bytes) return B200VIS_OK;
    if (ctx->h_edit) cudaFreeHost(ctx->h_edit);
    ctx->h_edit = nullptr; ctx->h_edit_bytes = 0;
    bytes = std::max<size_t>(bytes, (size_t)1 << 20);
    CU(cudaMallocHost(&ctx->h_edit, bytes));
    ctx->h_edit_bytes = bytes;
    return B200VIS_OK;
}

// The spare rank arrays an edit's rank merge and a compaction write into (swapped in when the call commits): each is
// allocated once, on first need, and assigned only when every array asked for was allocated, so a failed allocation
// leaves none of them half set up.  keys: also the spare of the resident keys.
static int32_t alloc_rank_spares(b200vis_ctx *ctx, bool keys) {
    const size_t N = ctx->cfg.max_entities;
    uint64_t *k = nullptr; uint32_t *r = nullptr, *rr = nullptr;
    cudaError_t e = cudaSuccess;
    if (keys && !ctx->d_keys2) e = dalloc(&k, N);
    if (e == cudaSuccess && !ctx->d_rank2) e = dalloc(&r, N);
    if (e == cudaSuccess && !ctx->d_row_of_rank2) e = dalloc(&rr, N);
    if (e != cudaSuccess) {
        cudaGetLastError();
        cudaFree(k); cudaFree(r); cudaFree(rr);
        return fail(ctx, e == cudaErrorMemoryAllocation ? B200VIS_ERR_OUT_OF_MEMORY : B200VIS_ERR_CUDA, "spare rank arrays: %s", cudaGetErrorString(e));
    }
    if (k) ctx->d_keys2 = k;
    if (r) ctx->d_rank2 = r;
    if (rr) ctx->d_row_of_rank2 = rr;
    return B200VIS_OK;
}

// Diff slots' sets (bit = rank) to new ranks: each slot that may hold entries (held), `sets` sets per slot, through the
// run's added / removed words (free between runs; they hold at least 2 * sets sets).  compacting: the set is cleared
// first, so words past the new end are empty.  A remapped slot's per-chunk counts (`count_sets` rows of them per slot)
// become "unknown" (non-zero), so that the next run reads every chunk of it.
static int32_t remap_slot_sets(b200vis_ctx *ctx, uint32_t *prev, uint32_t *prev_count, uint32_t *scratch, uint32_t sets, uint32_t count_sets,
                               const std::vector<uint8_t> &held, bool compacting, uint32_t n_words, uint32_t n_rows, uint32_t n_old_rows,
                               const uint32_t *row_of_rank, const uint32_t *old_rank) {
    cudaStream_t st = ctx->stream;
    const size_t ws = ctx->vis.words_stride, cs = ctx->vis.chunks_stride;
    for (uint32_t s = 0; s < held.size(); ++s) {
        if (!held[s]) continue;
        uint32_t *set = prev + (size_t)s * sets * ws;
        CU(cudaMemcpyAsync(scratch, set, sets * ws * 4, cudaMemcpyDeviceToDevice, st));
        if (compacting) CU(cudaMemsetAsync(set, 0, sets * ws * 4, st));
        launch_remap_rank_sets(st, scratch, set, (uint32_t)ws, sets, n_words, n_rows, n_old_rows, row_of_rank, old_rank);
        CU(cudaGetLastError());
        CU(cudaMemsetAsync(prev_count + (size_t)s * count_sets * cs, 0xFF, count_sets * cs * 4, st));
    }
    return B200VIS_OK;
}
// ... for the shadow diff's slots (six sets each) and the view diff's (eight sets each, one count row)
static int32_t remap_diff_slots(b200vis_ctx *ctx, bool compacting, uint32_t n_words, uint32_t n_rows, uint32_t n_old_rows,
                                const uint32_t *row_of_rank, const uint32_t *old_rank) {
    int32_t rc;
    if (ctx->sdiff.added &&
        (rc = remap_slot_sets(ctx, ctx->sdiff.prev, ctx->sdiff.prev_count, ctx->sdiff.words, 6, 6, ctx->sdiff_held, compacting, n_words,
                              n_rows, n_old_rows, row_of_rank, old_rank)))
        return rc;
    if (ctx->vdiff.added &&
        (rc = remap_slot_sets(ctx, ctx->vdiff.prev, ctx->vdiff.prev_count, ctx->vdiff.words, 8, 1, ctx->vdiff_held, compacting, n_words,
                              n_rows, n_old_rows, row_of_rank, old_rank)))
        return rc;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_edit_topology(b200vis_ctx *ctx, uint32_t n_despawn, const uint32_t *despawn_rows,
                                         uint32_t n_reparent, const uint32_t *reparent_rows, const uint32_t *new_parent,
                                         uint32_t n_spawn, const uint32_t *spawn_parent, const uint64_t *spawn_entity_bits) {
    CHECK_CTX_JOIN();   // the tail of the frame in flight reads the rank arrays and the visible sets
    if (!ctx->topology_set || !ctx->hplan) return fail(ctx, B200VIS_ERR_NOT_READY, "edit_topology: b200vis_set_topology has not been called");
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "edit_topology: world_size > 1 (use set_topology)");
    if ((n_despawn && !despawn_rows) || (n_reparent && (!reparent_rows || !new_parent)) || (n_spawn && (!spawn_parent || !spawn_entity_bits)))
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: null array");
    Plan &hp = *ctx->hplan;
    const uint32_t n = ctx->n, n2 = n + n_spawn;
    if ((uint64_t)n + n_spawn > ctx->cfg.max_entities)
        return fail(ctx, B200VIS_ERR_CAPACITY, "edit_topology: %u + %u rows exceed max_entities %u", n, n_spawn, ctx->cfg.max_entities);
    cudaStream_t st = ctx->stream;
    if (ctx->ev_edit) CU(cudaEventSynchronize(ctx->ev_edit));   // the last edit's staging copies have been read
    else CU(cudaEventCreateWithFlags(&ctx->ev_edit, cudaEventDisableTiming));
    // ---- ranks of the new keys: appended (rank == row stays true) or merged on the device ----
    std::vector<uint32_t> ord(n_spawn);
    std::iota(ord.begin(), ord.end(), 0u);
    std::sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return spawn_entity_bits[a] < spawn_entity_bits[b]; });
    for (uint32_t i = 1; i < n_spawn; ++i)
        if (spawn_entity_bits[ord[i]] == spawn_entity_bits[ord[i - 1]])
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: entity bits %llx spawned twice", (unsigned long long)spawn_entity_bits[ord[i]]);
    ctx->shadow_emit_ready = false;   // rows and rank order change: the last shadow run's bits name other entities
    bool append = ctx->rank_identity;
    for (uint32_t k = 0; k < n_spawn && append; ++k)
        append = k ? spawn_entity_bits[k] > spawn_entity_bits[k - 1] : (n == 0 || spawn_entity_bits[0] > ctx->max_key);
    const bool merge = n_spawn && !append;
    const size_t keys_off = 0, rows_off = (size_t)n_spawn * 8, dup_off = rows_off + (((size_t)n_spawn * 4 + 15) & ~(size_t)15);
    if (merge) {
        const size_t N = ctx->cfg.max_entities;
        if (!ctx->d_keys) CU(dalloc(&ctx->d_keys, N));
        { const int32_t arc = alloc_rank_spares(ctx, true); if (arc) return arc; }
        if (!ctx->keys_resident) {
            CU(cudaStreamSynchronize(st));
            CU(cudaMemcpy(ctx->d_keys, ctx->h_keys.data(), (size_t)n * 8, cudaMemcpyHostToDevice));
            ctx->keys_resident = true;
            std::vector<uint64_t>().swap(ctx->h_keys);
        }
        int32_t rc = grow_edit_staging(ctx, dup_off + 16); if (rc) return rc;
        uint64_t *hk = reinterpret_cast<uint64_t *>(ctx->h_edit + keys_off);
        uint32_t *hr = reinterpret_cast<uint32_t *>(ctx->h_edit + rows_off);
        uint32_t *hd = reinterpret_cast<uint32_t *>(ctx->h_edit + dup_off);
        for (uint32_t j = 0; j < n_spawn; ++j) { hk[j] = spawn_entity_bits[ord[j]]; hr[j] = n + ord[j]; }
        hd[0] = 0;
        if (dup_off + 4 > ctx->stage_bytes) return fail(ctx, B200VIS_ERR_CAPACITY, "staging buffer too small");
        CU(cudaMemcpyAsync(ctx->d_stage, ctx->h_edit, dup_off + 4, cudaMemcpyHostToDevice, st));
        uint32_t *d_dup = reinterpret_cast<uint32_t *>(ctx->d_stage + dup_off);
        launch_rank_merge(st, ctx->d_keys, ctx->rank_identity ? nullptr : ctx->d_row_of_rank, n,
                          reinterpret_cast<const uint64_t *>(ctx->d_stage + keys_off), reinterpret_cast<const uint32_t *>(ctx->d_stage + rows_off),
                          n_spawn, ctx->d_keys2, ctx->d_row_of_rank2, ctx->d_rank2, d_dup);
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(hd, d_dup, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (hd[0]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: a spawned entity's bits equal those of an existing (live or dead) row");
    }
    if (n_despawn && (ctx->lights.n || !ctx->h_shadow.empty())) {   // a dead row must not go on being clustered or shadowed
        std::vector<uint32_t> ds(despawn_rows, despawn_rows + n_despawn);
        std::sort(ds.begin(), ds.end());
        for (uint32_t i = 0; i < ctx->lights.n; ++i)
            if (std::binary_search(ds.begin(), ds.end(), ctx->h_light_row[i]))
                return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: row %u is light %u: remove it with b200vis_set_lights first", ctx->h_light_row[i], i);
        for (size_t i = 0; i < ctx->h_shadow.size(); ++i)
            if (ctx->h_shadow[i].kind != B200VIS_SHADOW_DIRECTIONAL_CASCADE && std::binary_search(ds.begin(), ds.end(), ctx->h_shadow[i].row))
                return fail(ctx, B200VIS_ERR_INVALID_ARG, "edit_topology: row %u is shadow item %zu: replace the shadow items first", ctx->h_shadow[i].row, i);
    }
    // ---- host plan ----
    if (hp.tiles_c.size() + n_spawn > ctx->tiles_cap) {
        // at most one new tile per spawned row.  Grown before the edit is validated, so the current plan is copied whole:
        // if the edit then fails, the next frame runs the unchanged plan from the new buffers
        const uint32_t cap = (uint32_t)std::max<size_t>(2 * (size_t)ctx->tiles_cap, hp.tiles_c.size() + n_spawn + 1024);
        Tile *t = nullptr; WarpTile *w = nullptr; uint8_t *s = nullptr;
        CU(dalloc(&t, cap)); CU(dalloc(&w, cap)); CU(dalloc(&s, (size_t)cap * kTileRows));
        CU(cudaMemcpyAsync(t, ctx->d_tiles, hp.tiles.size() * sizeof(Tile), cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(w, ctx->d_wtiles, hp.wtiles.size() * sizeof(WarpTile), cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(s, ctx->d_sched, hp.tiles_c.size() * (size_t)kTileRows, cudaMemcpyDeviceToDevice, st));
        CU(cudaStreamSynchronize(st));
        cudaFree(ctx->d_tiles); cudaFree(ctx->d_wtiles); cudaFree(ctx->d_sched);
        ctx->d_tiles = t; ctx->d_wtiles = w; ctx->d_sched = s; ctx->tiles_cap = cap;
    }
    const TopologyEdit ed{n_despawn, despawn_rows, n_reparent, reparent_rows, new_parent, n_spawn, spawn_parent};
    EditResult er;
    int32_t rc = edit_plan(ctx, hp, ctx->cfg.max_entities, ed, er);
    if (rc) return rc;
    // ---- commit: one pinned staging packet, async copies of the descriptors, the re-planned rows and schedule blocks ----
    const size_t T = hp.tiles.size();
    size_t bytes = T * (sizeof(Tile) + sizeof(WarpTile)) + (size_t)er.rows * 12 + er.tiles.size() * (size_t)kTileRows +
                   ((size_t)n_despawn + n_reparent) * 4 + (append ? (size_t)n_spawn * 8 : 0) + 64;
    rc = grow_edit_staging(ctx, bytes); if (rc) return rc;
    uint8_t *h = ctx->h_edit;
    size_t off = 0;
    auto put = [&](void *dst, const void *src, size_t nb) -> int32_t {
        if (!nb) return B200VIS_OK;
        memcpy(h + off, src, nb);
        CU(cudaMemcpyAsync(dst, h + off, nb, cudaMemcpyHostToDevice, st));
        off += (nb + 15) & ~(size_t)15;
        return B200VIS_OK;
    };
    if ((rc = put(ctx->d_tiles, hp.tiles.data(), T * sizeof(Tile)))) return rc;
    if ((rc = reset_tile_hints(ctx, st))) return rc;
    if ((rc = put(ctx->d_wtiles, hp.wtiles.data(), T * sizeof(WarpTile)))) return rc;
    for (const auto &rg : er.ranges) {
        const size_t a = rg.first, c = (size_t)(rg.second - rg.first) * 4;
        if ((rc = put(ctx->rows.topo + a, hp.topo.data() + a, c))) return rc;
        if ((rc = put(ctx->d_wtopo + a, hp.wtopo.data() + a, c))) return rc;
        if ((rc = put(ctx->d_parent + a, hp.parent.data() + a, c))) return rc;
    }
    for (uint32_t ci : er.tiles)
        if ((rc = put(ctx->d_sched + (size_t)ci * kTileRows, hp.sched.data() + (size_t)ci * kTileRows, kTileRows))) return rc;
    // row lists of the column kernel: through the device staging buffer (stream-ordered after the merge that used it)
    const size_t lists = ((size_t)n_despawn + n_reparent) * 4;
    if (lists > ctx->stage_bytes) return fail(ctx, B200VIS_ERR_CAPACITY, "staging buffer too small");
    if ((rc = put(ctx->d_stage, despawn_rows, (size_t)n_despawn * 4))) return rc;
    if ((rc = put(ctx->d_stage + (size_t)n_despawn * 4, reparent_rows, (size_t)n_reparent * 4))) return rc;
    CU(cudaEventRecord(ctx->ev_edit, st));
    RowEdit re{};
    re.dead = reinterpret_cast<const uint32_t *>(ctx->d_stage); re.n_dead = n_despawn;
    re.moved = reinterpret_cast<const uint32_t *>(ctx->d_stage + (size_t)n_despawn * 4); re.n_moved = n_reparent;
    re.first_new = n; re.n_new = n_spawn;
    re.cls = ctx->d_cls; re.caster = ctx->d_caster; re.visibility = ctx->d_visibility; re.vv_shadow = ctx->d_vv_shadow;
    re.layers = ctx->have_layers ? ctx->d_layers : nullptr; re.layers_ext = ctx->d_layers_ext;
    re.range = ctx->have_range ? ctx->d_range : nullptr; re.range_se = ctx->d_range_se; re.range_ua = ctx->d_range_ua;
    Rows R = ctx->rows;
    launch_edit_rows(st, R, re);
    CU(cudaGetLastError());
    // ---- ranks ----
    if (merge) {
        const uint32_t *old_rank = ctx->rank_identity ? nullptr : ctx->d_rank;
        std::swap(ctx->d_keys, ctx->d_keys2); std::swap(ctx->d_rank, ctx->d_rank2); std::swap(ctx->d_row_of_rank, ctx->d_row_of_rank2);
        if (ctx->diff.prev) {   // last frame's visible sets, bit = rank: to the new ranks (diff.words is free between frames)
            const size_t words = (size_t)ctx->vis.words_stride * ctx->cfg.max_views;
            CU(cudaMemcpyAsync(ctx->diff.words, ctx->diff.prev, words * 4, cudaMemcpyDeviceToDevice, st));
            launch_remap_rank_sets(st, ctx->diff.words, ctx->diff.prev, ctx->vis.words_stride, ctx->cfg.max_views, (n2 + 31) / 32, n2, n,
                                   ctx->d_row_of_rank, old_rank);
            CU(cudaGetLastError());
        }
        if ((rc = remap_diff_slots(ctx, false, (n2 + 31) / 32, n2, n, ctx->d_row_of_rank, old_rank))) return rc;
        ctx->rank_identity = false;
    } else if (n_spawn) {
        if (ctx->keys_resident) { if ((rc = put(ctx->d_keys + n, spawn_entity_bits, (size_t)n_spawn * 8))) return rc; CU(cudaEventRecord(ctx->ev_edit, st)); }
        else ctx->h_keys.insert(ctx->h_keys.end(), spawn_entity_bits, spawn_entity_bits + n_spawn);
    }
    if (n_spawn) ctx->max_key = std::max(ctx->max_key, spawn_entity_bits[ord[n_spawn - 1]]);
    install_passes(ctx, hp);
    ctx->n = n2;
    ctx->rows.n = n2;
    ctx->vis.n_words = (n2 + 31) / 32;
    // the visible masks are empty between frames and the chunk counters past the old row count were never written: growing
    // n_words / n_chunks needs no clearing
    ctx->vis.n_chunks = (ctx->vis.n_words + kChunkWords - 1) / kChunkWords;
    ctx->gt_aos_valid = false;
    return tables_unmap_rows(ctx, n_despawn, despawn_rows);
}

extern "C" int32_t b200vis_compact_topology(b200vis_ctx *ctx, uint32_t n_reparent, const uint32_t *reparent_rows,
                                            const uint32_t *new_parent, uint32_t *old_to_new_out) {
    CHECK_CTX_JOIN();   // the tail of the frame in flight writes the lists and reads the rank arrays
    if (!ctx->topology_set || !ctx->hplan) return fail(ctx, B200VIS_ERR_NOT_READY, "compact_topology: b200vis_set_topology has not been called");
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "compact_topology: world_size > 1 (use set_topology)");
    if (n_reparent && (!reparent_rows || !new_parent)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "compact_topology: null array");
    ctx->shadow_emit_ready = false;   // rows and rank order change: the last shadow run's bits name other entities
    Plan &hp = *ctx->hplan;
    const uint32_t n = ctx->n, V = ctx->cfg.max_views;
    cudaStream_t st = ctx->stream;
    if (ctx->ev_edit) CU(cudaEventSynchronize(ctx->ev_edit));   // the last edit's staging copies have been read
    else CU(cudaEventCreateWithFlags(&ctx->ev_edit, cudaEventDisableTiming));
    // ---- the row-valued results the context holds: every view slot's visible list (an inactive view keeps its last
    // one), the visible diff, the shadow lists.  A dead row they name survives this compaction as a tombstone ----
    // the visible-diff state exists once the diff was ever enabled, and stays what the shadow stage reads and what a
    // download returns even while the diff is switched off: it is carried over whenever it exists, as the edit does
    const bool diff = ctx->diff.prev != nullptr;
    const uint32_t LS = ctx->vis.list_stride;
    RowLists lists[4]; uint32_t n_lists = 0;
    lists[n_lists++] = RowLists{ctx->vis.lists, LS, V, 1, reinterpret_cast<const uint32_t *>(ctx->d_stats)};   // DevStats::visible_count
    if (diff) {
        lists[n_lists++] = RowLists{ctx->diff.lists, LS, V, 2, ctx->diff.count};                        // added
        lists[n_lists++] = RowLists{ctx->diff.lists + (size_t)V * LS, LS, V, 2, ctx->diff.count + 1};   // removed
    }
    if (ctx->shadow.n_lights) lists[n_lists++] = RowLists{ctx->shadow.lists, ctx->shadow.list_cap, ctx->shadow.n_lights * 6, 1, ctx->shadow.count};
    // what the call allocates for itself only (scratch for small worlds, trace events): released on every return
    struct CallScratch {
        uint8_t *tmp = nullptr; cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
        ~CallScratch() { if (tmp) cudaFree(tmp); for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
    } own;
    std::vector<uint32_t> held;
    if (hp.n_dead) {
        CU(cudaMemsetAsync(ctx->d_dirty, 0, n, st));
        for (uint32_t i = 0; i < n_lists; ++i) launch_mark_listed_rows(st, lists[i], n, ctx->d_dirty, n);
        if (diff)   // last frame's visible sets: a row in them is reported removed by the next diff
            launch_mark_set_rows(st, ctx->diff.prev, ctx->vis.words_stride, V, (n + 31) / 32, ctx->rank_identity ? nullptr : ctx->d_row_of_rank, ctx->d_dirty);
        if (ctx->sdiff.added)   // ... and the shadow diff slots' sets, likewise
            for (uint32_t s = 0; s < ctx->sdiff_max_slots; ++s)
                if (ctx->sdiff_held[s])
                    launch_mark_set_rows(st, ctx->sdiff.prev + (size_t)s * 6 * ctx->vis.words_stride, ctx->vis.words_stride, 6, (n + 31) / 32,
                                         ctx->rank_identity ? nullptr : ctx->d_row_of_rank, ctx->d_dirty);
        if (ctx->vdiff.added)   // ... and the view diff slots' sets
            for (uint32_t s = 0; s < ctx->vdiff_max_slots; ++s)
                if (ctx->vdiff_held[s])
                    launch_mark_set_rows(st, ctx->vdiff.prev + (size_t)s * 8 * ctx->vis.words_stride, ctx->vis.words_stride, 8, (n + 31) / 32,
                                         ctx->rank_identity ? nullptr : ctx->d_row_of_rank, ctx->d_dirty);
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(ctx->h_stage, ctx->d_dirty, n, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        for (uint32_t r = 0; r < n; ++r) if (!hp.alive[r] && ctx->h_stage[r]) held.push_back(r);
    }
    // ---- host plan (validates everything; nothing is changed before it succeeds) ----
    // B200VIS_COMPACT_TRACE: host clock around the planning, events around the device work, one line on stderr per call
    static int trace = -1;
    if (trace < 0) trace = getenv("B200VIS_COMPACT_TRACE") ? 1 : 0;
    using clk = std::chrono::steady_clock;
    const auto t_plan0 = clk::now();
    Plan q;
    std::vector<uint32_t> o2n, n2o;
    int32_t rc = compact_plan(ctx, hp, n_reparent, reparent_rows, new_parent, held, 0, q, o2n, n2o);
    if (rc) return rc;
    const double plan_ms = std::chrono::duration<double, std::milli>(clk::now() - t_plan0).count();
    cudaEvent_t *tev = own.ev;
    float gather_ms = 0.f, copy_ms = 0.f;
    size_t row_bytes = 0;
    if (trace) for (int i = 0; i < 3; ++i) CU(cudaEventCreate(&tev[i]));
    const uint32_t n2 = (uint32_t)n2o.size(), T = (uint32_t)q.tiles.size();
    std::vector<uint32_t> dropped;
    for (uint32_t r = 0; r < n; ++r) if (o2n[r] == kNoParent) dropped.push_back(r);
    const uint32_t nd = (uint32_t)dropped.size();
    // ---- the resident per-row columns the permutation moves (columns never uploaded are absent) ----
    struct Column { void *p; uint32_t elem, per_row; unsigned long long fill; };   // fill: value of the rows past the new count
    std::vector<Column> cols;
    {
        auto add = [&](void *p, uint32_t elem, uint32_t per_row, unsigned long long fill) { if (p) cols.push_back(Column{p, elem, per_row, fill}); };
        const Rows &R = ctx->rows;
        for (void *p : {(void *)R.trsA, (void *)R.trsB, (void *)R.gt0, (void *)R.gt1, (void *)R.gt2, (void *)R.bndA}) add(p, 16, 1, 0);
        add(R.trsC, 8, 1, 0); add(R.bndB, 8, 1, 0);
        add(ctx->d_layers_ext, 8, 3, 0);                                   // RenderLayers blocks 1..3
        if (ctx->have_layers) add(ctx->d_layers, 8, 1, 1);                 // block 0; RenderLayers::default()
        add(ctx->d_range_se, 8, 1, 0);
        if (ctx->have_range) add(ctx->d_range, 4, 1, 0);
        add(ctx->d_light_ord, 4, 1, 0xFFFFFFFFull);                        // not a light
        for (void *p : {(void *)R.flags, (void *)R.state, (void *)ctx->d_cls, (void *)ctx->d_range_ua, (void *)ctx->d_visibility,
                        (void *)ctx->d_iv_changed, (void *)ctx->d_caster}) add(p, 1, 1, 0);
        add(ctx->d_vv_shadow, 1, 1, 0xFF);                                 // the host's value unknown
        add(ctx->d_tvv_shadow, 1, 1, 0xFF);                                // the same for the table write-back
    }
    // ---- device scratch: the maps, then the permuted columns (a group at a time) and the reparented rows ----
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t o_o2n = 0, o_n2o = al((size_t)n * 4), o_drow = o_n2o + al((size_t)n2 * 4), o_drk = o_drow + al((size_t)nd * 4),
                 o_src = o_drk + al((size_t)nd * 4), o_flag = o_src + al((size_t)n2 * 4), o_cols = o_flag + 256;
    size_t max_col = al((size_t)n_reparent * 4), all_cols = max_col;
    for (const Column &c : cols) { const size_t nb = al((size_t)n * c.elem * c.per_row); max_col = std::max(max_col, nb); all_cols += nb; }
    // ---- buffers, all before the first device write (a failed allocation leaves the world as it was) ----
    if ((rc = alloc_rank_spares(ctx, ctx->keys_resident))) return rc;
    const uint32_t n_items = ctx->shadow.n_lights;
    const size_t bytes = ((size_t)n + 2 * n2 + 2 * nd + ctx->lights.n + n_reparent) * 4 + (size_t)n_items * sizeof(ShadowLight) + (size_t)n2 * 12 +
                         (size_t)T * (sizeof(Tile) + sizeof(WarpTile) + kTileRows) + 16 * 16 + 64;
    if ((rc = grow_edit_staging(ctx, bytes))) return rc;
    uint8_t *scratch = ctx->d_stage;
    size_t scratch_bytes = ctx->stage_bytes;
    if (o_cols + max_col > scratch_bytes) {
        // a small world: its 64 B/row staging buffer cannot hold the maps' aligned regions next to the widest column.  A
        // scratch buffer of its own for this call, large enough for every column in one group
        scratch_bytes = o_cols + all_cols;
        const cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&own.tmp), scratch_bytes);
        if (e != cudaSuccess) {
            cudaGetLastError(); own.tmp = nullptr;
            return fail(ctx, B200VIS_ERR_OUT_OF_MEMORY, "compact_topology: %zu bytes of scratch: %s", scratch_bytes, cudaGetErrorString(e));
        }
        scratch = own.tmp;
    }
    if (T > ctx->tiles_cap) {
        const uint32_t cap = T + 1024;
        Tile *t = nullptr; WarpTile *w = nullptr; uint8_t *s = nullptr;
        if (dalloc(&t, cap) != cudaSuccess || dalloc(&w, cap) != cudaSuccess || dalloc(&s, (size_t)cap * kTileRows) != cudaSuccess) {
            cudaGetLastError();
            if (t) cudaFree(t); if (w) cudaFree(w); if (s) cudaFree(s);
            return fail(ctx, B200VIS_ERR_OUT_OF_MEMORY, "compact_topology: tile descriptors for %u tiles", T);
        }
        CU(cudaStreamSynchronize(st));
        cudaFree(ctx->d_tiles); cudaFree(ctx->d_wtiles); cudaFree(ctx->d_sched);
        ctx->d_tiles = t; ctx->d_wtiles = w; ctx->d_sched = s; ctx->tiles_cap = cap;
    }
    uint32_t *d_o2n = reinterpret_cast<uint32_t *>(scratch + o_o2n), *d_n2o = reinterpret_cast<uint32_t *>(scratch + o_n2o);
    uint32_t *d_drow = reinterpret_cast<uint32_t *>(scratch + o_drow), *d_drk = reinterpret_cast<uint32_t *>(scratch + o_drk);
    uint32_t *d_src = reinterpret_cast<uint32_t *>(scratch + o_src), *d_flag = reinterpret_cast<uint32_t *>(scratch + o_flag);
    uint8_t *h = ctx->h_edit;
    size_t off = 0;
    auto put = [&](void *dst, const void *src, size_t nb) -> int32_t {
        if (!nb) return B200VIS_OK;
        memcpy(h + off, src, nb);
        CU(cudaMemcpyAsync(dst, h + off, nb, cudaMemcpyHostToDevice, st));
        off += (nb + 15) & ~(size_t)15;
        return B200VIS_OK;
    };
    const auto t_dev0 = clk::now();
    if ((rc = put(d_o2n, o2n.data(), (size_t)n * 4))) return rc;
    if ((rc = put(d_n2o, n2o.data(), (size_t)n2 * 4))) return rc;
    // ---- ranks: the dropped rows' keys go, every other rank moves down by the dropped ranks below it ----
    std::vector<uint32_t> drk;
    if (ctx->rank_identity) drk = dropped;
    else if (nd) {
        if ((rc = put(d_drow, dropped.data(), (size_t)nd * 4))) return rc;
        launch_gather_u32(st, ctx->d_rank, d_drow, nd, d_drk);
        CU(cudaGetLastError());
        drk.resize(nd);
        CU(cudaMemcpyAsync(ctx->h_stage, d_drk, (size_t)nd * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        memcpy(drk.data(), ctx->h_stage, (size_t)nd * 4);
        std::sort(drk.begin(), drk.end());
    }
    if ((rc = put(d_drk, drk.data(), (size_t)nd * 4))) return rc;
    CU(cudaMemsetAsync(d_flag, 0, 4, st));
    launch_compact_ranks(st, ctx->rank_identity ? nullptr : ctx->d_row_of_rank, ctx->keys_resident ? ctx->d_keys : nullptr, n, d_drk, nd, d_o2n,
                         ctx->d_row_of_rank2, ctx->d_rank2, ctx->keys_resident ? ctx->d_keys2 : nullptr, d_src, d_flag);
    CU(cudaGetLastError());
    // last frame's visible sets (bit = rank) to the new ranks, through diff.words (free between frames); words past the new
    // end cleared
    if (diff) {
        const size_t words = (size_t)ctx->vis.words_stride * V;
        CU(cudaMemcpyAsync(ctx->diff.words, ctx->diff.prev, words * 4, cudaMemcpyDeviceToDevice, st));
        CU(cudaMemsetAsync(ctx->diff.prev, 0, words * 4, st));
        launch_remap_rank_sets(st, ctx->diff.words, ctx->diff.prev, ctx->vis.words_stride, V, (n2 + 31) / 32, n2, n, d_src, nullptr);
        CU(cudaGetLastError());
    }
    if ((rc = remap_diff_slots(ctx, true, (n2 + 31) / 32, n2, n, d_src, nullptr))) return rc;
    // ---- the lists results hold, renumbered in place (survivors keep their rank order, so every list stays sorted) ----
    for (uint32_t i = 0; i < n_lists; ++i) launch_renumber_listed_rows(st, lists[i], n, d_o2n, n);
    if ((rc = flush_table_updates(ctx))) return rc;      // queued map updates carry the old row numbers
    if (ctx->tables_set && !ctx->h_tab_map.empty()) {   // the tables' slot -> row maps: mapped rows are live, none is dropped
        const uint32_t slots = (uint32_t)ctx->h_tab_map.size();
        launch_renumber_listed_rows(st, RowLists{ctx->d_tab_map, slots, 1, 1, ctx->d_tab_total}, slots, d_o2n, n);
    }
    CU(cudaGetLastError());
    // ---- the row permutation of every resident per-row column, in groups that fit the staging buffer ----
    {
        RowPermute pm{};
        pm.new_to_old = d_n2o; pm.n_new = n2; pm.n_old = n;
        void *home[kPermuteCols];
        const size_t avail = scratch_bytes - o_cols;   // >= the widest column (checked before the first write)
        size_t used = 0;
        auto flush = [&]() -> int32_t {
            if (!pm.n_cols) return B200VIS_OK;
            if (trace) CU(cudaEventRecord(tev[0], st));
            launch_permute_rows(st, pm);
            CU(cudaGetLastError());
            if (trace) CU(cudaEventRecord(tev[1], st));
            for (uint32_t c = 0; c < pm.n_cols; ++c) {
                CU(cudaMemcpyAsync(home[c], pm.col[c].dst, (size_t)n * pm.col[c].elem * pm.col[c].per_row, cudaMemcpyDeviceToDevice, st));
                row_bytes += (size_t)pm.col[c].elem * pm.col[c].per_row;
            }
            if (trace) {
                float a = 0.f, b = 0.f;
                CU(cudaEventRecord(tev[2], st));
                CU(cudaEventSynchronize(tev[2]));
                CU(cudaEventElapsedTime(&a, tev[0], tev[1])); CU(cudaEventElapsedTime(&b, tev[1], tev[2]));
                gather_ms += a; copy_ms += b;
            }
            pm.n_cols = 0; used = 0;
            return B200VIS_OK;
        };
        for (const Column &c : cols) {
            const size_t nb = al((size_t)n * c.elem * c.per_row);
            if (used + nb > avail || pm.n_cols == (uint32_t)kPermuteCols) { if ((rc = flush())) return rc; }
            home[pm.n_cols] = c.p;
            pm.col[pm.n_cols++] = PermuteColumn{c.p, scratch + o_cols + used, c.elem, c.per_row, c.fill};
            used += nb;
        }
        if ((rc = flush())) return rc;
    }
    if (n_reparent) {   // Changed<ChildOf> / RemovedComponents<ChildOf>: marked as the reparent step of edit_topology marks them
        std::vector<uint32_t> moved(n_reparent);
        for (uint32_t j = 0; j < n_reparent; ++j) moved[j] = o2n[reparent_rows[j]];
        uint32_t *d_moved = reinterpret_cast<uint32_t *>(scratch + o_cols);
        if ((rc = put(d_moved, moved.data(), (size_t)n_reparent * 4))) return rc;
        RowEdit re{};
        re.moved = d_moved; re.n_moved = n_reparent;
        launch_edit_rows(st, ctx->rows, re);
        CU(cudaGetLastError());
    }
    // ---- light and shadow-item rows (ordinals and item order unchanged), the plan, the state past the new end ----
    for (uint32_t &r : ctx->h_light_row) if (r < n) r = o2n[r];   // a light is never a dead row
    if ((rc = put(ctx->d_light_row, ctx->h_light_row.data(), (size_t)ctx->lights.n * 4))) return rc;
    for (ShadowLight &s : ctx->h_shadow) if (s.kind != B200VIS_SHADOW_DIRECTIONAL_CASCADE) s.row = o2n[s.row];
    if ((rc = put(ctx->d_shadow_lights, ctx->h_shadow.data(), (size_t)n_items * sizeof(ShadowLight)))) return rc;
    if ((rc = put(ctx->rows.topo, q.topo.data(), (size_t)n2 * 4))) return rc;
    if ((rc = put(ctx->d_wtopo, q.wtopo.data(), (size_t)n2 * 4))) return rc;
    if ((rc = put(ctx->d_parent, q.parent.data(), (size_t)n2 * 4))) return rc;
    if ((rc = put(ctx->d_tiles, q.tiles.data(), (size_t)T * sizeof(Tile)))) return rc;
    if ((rc = reset_tile_hints(ctx, st))) return rc;
    if ((rc = put(ctx->d_wtiles, q.wtiles.data(), (size_t)T * sizeof(WarpTile)))) return rc;
    if ((rc = put(ctx->d_sched, q.sched.data(), q.sched.size()))) return rc;
    CU(cudaEventRecord(ctx->ev_edit, st));
    const uint32_t nw2 = (n2 + 31) / 32, nc2 = (nw2 + kChunkWords - 1) / kChunkWords;
    {   // growing the row count later relies on every mask word and chunk counter past the count being zero
        const VisibleBufs &vb = ctx->vis;
        if (vb.words_stride > nw2) CU(cudaMemset2DAsync(vb.mask + nw2, (size_t)vb.words_stride * 4, 0, (size_t)(vb.words_stride - nw2) * 4, 2 * V, st));
        if (vb.chunks_stride > nc2) {
            CU(cudaMemset2DAsync(vb.chunk_count + nc2, (size_t)vb.chunks_stride * 4, 0, (size_t)(vb.chunks_stride - nc2) * 4, 3 * kMaxCameras, st));
            if (ctx->diff.chunk) CU(cudaMemset2DAsync(ctx->diff.chunk + nc2, (size_t)vb.chunks_stride * 4, 0, (size_t)(vb.chunks_stride - nc2) * 4, V, st));
            if (ctx->shadow.chunk_count)
                CU(cudaMemset2DAsync(ctx->shadow.chunk_count + nc2, (size_t)vb.chunks_stride * 4, 0, (size_t)(vb.chunks_stride - nc2) * 4,
                                     (size_t)ctx->shadow_cap_lights * 6, st));
        }
    }
    uint32_t *h_flag = reinterpret_cast<uint32_t *>(h + off);
    CU(cudaMemcpyAsync(h_flag, d_flag, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    // ---- commit ----
    std::swap(ctx->d_rank, ctx->d_rank2); std::swap(ctx->d_row_of_rank, ctx->d_row_of_rank2);
    if (ctx->keys_resident) std::swap(ctx->d_keys, ctx->d_keys2);
    else {
        std::vector<uint64_t> keys; keys.reserve(n2);
        for (uint32_t rk = 0, j = 0; rk < n; ++rk) { if (j < nd && drk[j] == rk) { ++j; continue; } keys.push_back(ctx->h_keys[rk]); }
        ctx->h_keys.swap(keys);
    }
    ctx->rank_identity = *h_flag == 0;
    *ctx->hplan = std::move(q);
    install_passes(ctx, *ctx->hplan);
    ctx->n = n2;
    ctx->rows.n = n2;
    ctx->vis.n_words = nw2;
    ctx->vis.n_chunks = nc2;
    ctx->gt_aos_valid = false;
    tables_renumber(ctx, o2n);
    if (old_to_new_out) memcpy(old_to_new_out, o2n.data(), (size_t)n * 4);
    if (trace) {
        const double dev_ms = std::chrono::duration<double, std::milli>(clk::now() - t_dev0).count();
        fprintf(stderr, "[b200vis_compact] rows %u -> %u (held %zu)  host plan %.3f ms  device part %.3f ms (host clock)  "
                "permute: %zu B/row, gather %.3f ms, copy-back %.3f ms\n",
                n, n2, held.size(), plan_ms, dev_ms, row_bytes, gather_ms, copy_ms);
    }
    return B200VIS_OK;
}

extern "C" int32_t b200vis_topology_summary(const b200vis_ctx *ctx, uint32_t out[4]) {
    if (!ctx || !out) return B200VIS_ERR_INVALID_ARG;
    const Plan *hp = ctx->hplan;
    out[0] = ctx->n;
    out[1] = hp ? ctx->n - hp->n_dead : ctx->n;
    out[2] = hp ? (uint32_t)hp->tiles.size() : 0u;
    out[3] = ctx->pass_begin.empty() ? 0u : (uint32_t)ctx->pass_begin.size() - 1;
    return B200VIS_OK;
}

// True when `row` is a despawned row (b200vis_edit_topology) that no compaction has dropped yet.
static bool row_is_dead(const b200vis_ctx *ctx, uint32_t row) {
    return ctx->hplan && row < ctx->hplan->n && !ctx->hplan->alive[row];
}

extern "C" int32_t b200vis_host_edit_plan(uint32_t n, const uint32_t *parent, uint32_t tile_rows, uint32_t max_rows, uint32_t script_words,
                                          const uint32_t *script, uint32_t tiles_capacity, uint32_t *n_rows_out, uint32_t *n_tiles,
                                          uint32_t *tile_desc, uint32_t *topo, uint32_t *wtopo, uint8_t *sched, uint32_t counters[4]) {
    if ((n && !parent) || (script_words && !script) || !n_rows_out || !n_tiles || !counters) return B200VIS_ERR_INVALID_ARG;
    Plan plan;
    int32_t rc = build_plan(nullptr, n, parent, tile_rows ? tile_rows : kTileRows, plan);
    if (rc) return rc;
    plan.parent.assign(parent, parent + n); plan.alive.assign(n, 1);
    counters[0] = counters[1] = counters[3] = 0;
    for (uint32_t at = 0; at < script_words;) {
        if (script_words - at < 3) { rc = fail(nullptr, B200VIS_ERR_INVALID_ARG, "host_edit_plan: truncated step header"); break; }
        if (script[at] == 0xFFFFFFFFu) {   // compaction step
            const uint32_t nr = script[at + 1], nh = script[at + 2];
            const uint64_t len = 3ull + 2ull * nr + nh;
            if (len > script_words - at) { rc = fail(nullptr, B200VIS_ERR_INVALID_ARG, "host_edit_plan: truncated step"); break; }
            const uint32_t *a = script + at + 3;
            const std::vector<uint32_t> held(a + 2 * nr, a + 2 * nr + nh);
            Plan q;
            std::vector<uint32_t> o2n, n2o;
            rc = compact_plan(nullptr, plan, nr, a, a + nr, held, tile_rows, q, o2n, n2o);
            if (rc) break;
            plan = std::move(q);
            counters[0] = (uint32_t)plan.tiles.size(); counters[1] = plan.n; counters[3]++;
            at += (uint32_t)len;
            continue;
        }
        const uint32_t nd = script[at], nr = script[at + 1], ns = script[at + 2];
        const uint64_t len = 3ull + nd + 2ull * nr + ns;
        if (len > script_words - at) { rc = fail(nullptr, B200VIS_ERR_INVALID_ARG, "host_edit_plan: truncated step"); break; }
        const uint32_t *a = script + at + 3;
        const TopologyEdit ed{nd, a, nr, a + nd, a + nd + nr, ns, a + nd + 2 * nr};
        EditResult er;
        rc = edit_plan(nullptr, plan, max_rows, ed, er);
        if (rc) break;
        counters[0] = (uint32_t)er.tiles.size(); counters[1] = er.rows; counters[3]++;
        at += (uint32_t)len;
    }
    counters[2] = plan.pass_begin.empty() ? 0u : (uint32_t)plan.pass_begin.size() - 1;
    *n_rows_out = plan.n;
    *n_tiles = (uint32_t)plan.tiles.size();
    if (!tile_desc) return rc;
    if (plan.tiles.size() > tiles_capacity || (plan.n && (!topo || !wtopo)) || !sched) return B200VIS_ERR_CAPACITY;
    for (size_t p = 0; p + 1 < plan.pass_begin.size(); ++p)
        for (uint32_t i = plan.pass_begin[p]; i < plan.pass_begin[p + 1]; ++i) {
            const Tile &t = plan.tiles[i];
            const WarpTile &w = plan.wtiles[i];
            uint32_t *d = tile_desc + (size_t)i * 17;
            d[0] = t.base; d[1] = t.n_rows; d[2] = t.n_levels; d[3] = t.warp_sync_mask; d[4] = t.top_levels;
            d[5] = (uint32_t)t.lvl_warps; d[6] = (uint32_t)(t.lvl_warps >> 32); d[7] = (uint32_t)p;
            d[8] = w.n_chunks | ((uint32_t)w.contig << 8);
            memcpy(d + 9, w.nonroot, sizeof w.nonroot);
            memcpy(sched + (size_t)i * kTileRows, plan.sched.data() + (size_t)w.sched * kTileRows, kTileRows);
        }
    if (plan.n) { memcpy(topo, plan.topo.data(), (size_t)plan.n * 4); memcpy(wtopo, plan.wtopo.data(), (size_t)plan.n * 4); }
    return rc;
}

extern "C" int32_t b200vis_host_plan_summary(uint32_t n, const uint32_t *parent, uint32_t out[4]) {
    if ((n && !parent) || !out) return B200VIS_ERR_INVALID_ARG;
    Plan plan;
    const int32_t rc = build_plan(nullptr, n, parent, kTileRows, plan);
    if (rc) return rc;
    std::vector<uint32_t> &topo = plan.topo, &pass_begin = plan.pass_begin; std::vector<Tile> &tiles = plan.tiles;
    uint32_t max_levels = 0, ext = 0;
    for (const Tile &t : tiles) max_levels = std::max<uint32_t>(max_levels, t.n_levels);
    for (uint32_t w : topo) ext += (w & T_EXT_PARENT) ? 1u : 0u;
    out[0] = (uint32_t)tiles.size(); out[1] = pass_begin.empty() ? 0u : (uint32_t)pass_begin.size() - 1; out[2] = max_levels; out[3] = ext;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_host_warp_plan(uint32_t n, const uint32_t *parent, uint32_t tile_rows, uint32_t tiles_capacity, uint32_t *n_tiles,
                                          uint32_t *tile_desc, uint32_t *nonroot, uint8_t *sched, uint32_t *wtopo) {
    if ((n && !parent) || !n_tiles) return B200VIS_ERR_INVALID_ARG;
    Plan plan;
    const int32_t rc = build_plan(nullptr, n, parent, tile_rows ? tile_rows : kTileRows, plan);
    if (rc) return rc;
    *n_tiles = (uint32_t)plan.wtiles.size();
    if (!tile_desc) return B200VIS_OK;
    if (plan.wtiles.size() > tiles_capacity || !nonroot || !sched || (n && !wtopo)) return B200VIS_ERR_CAPACITY;
    std::vector<uint32_t> pass_of(plan.wtiles.size(), 0);
    for (size_t p = 0; p + 1 < plan.pass_begin.size(); ++p)
        for (uint32_t i = plan.pass_begin[p]; i < plan.pass_begin[p + 1]; ++i) pass_of[i] = (uint32_t)p;
    for (size_t i = 0; i < plan.wtiles.size(); ++i) {
        const WarpTile &w = plan.wtiles[i];
        tile_desc[i * 4 + 0] = w.base; tile_desc[i * 4 + 1] = w.n_rows;
        tile_desc[i * 4 + 2] = w.n_chunks | ((uint32_t)w.contig << 8); tile_desc[i * 4 + 3] = pass_of[i];
        memcpy(nonroot + i * kWarpChunks, w.nonroot, sizeof w.nonroot);
        memcpy(sched + i * (size_t)kTileRows, plan.sched.data() + (size_t)w.sched * kTileRows, kTileRows);
    }
    if (n) memcpy(wtopo, plan.wtopo.data(), (size_t)n * 4);
    return B200VIS_OK;
}

extern "C" int32_t b200vis_host_tile_plan(uint32_t n, const uint32_t *parent, uint32_t tile_rows, uint32_t tiles_capacity, uint32_t *n_tiles,
                                          uint32_t *tile_desc, uint32_t *topo) {
    if ((n && !parent) || !n_tiles) return B200VIS_ERR_INVALID_ARG;
    Plan plan;
    const int32_t rc = build_plan(nullptr, n, parent, tile_rows ? tile_rows : kTileRows, plan);
    if (rc) return rc;
    *n_tiles = (uint32_t)plan.tiles.size();
    if (!tile_desc) return B200VIS_OK;
    if (plan.tiles.size() > tiles_capacity || (n && !topo)) return B200VIS_ERR_CAPACITY;
    std::vector<uint32_t> pass_of(plan.tiles.size(), 0);
    for (size_t p = 0; p + 1 < plan.pass_begin.size(); ++p)
        for (uint32_t i = plan.pass_begin[p]; i < plan.pass_begin[p + 1]; ++i) pass_of[i] = (uint32_t)p;
    for (size_t i = 0; i < plan.tiles.size(); ++i) {
        const Tile &t = plan.tiles[i];
        uint32_t *d = tile_desc + i * 8;
        d[0] = t.base; d[1] = t.n_rows; d[2] = t.n_levels; d[3] = t.warp_sync_mask; d[4] = t.top_levels;
        d[5] = (uint32_t)t.lvl_warps; d[6] = (uint32_t)(t.lvl_warps >> 32); d[7] = pass_of[i];
    }
    if (n) memcpy(topo, plan.topo.data(), (size_t)n * 4);
    return B200VIS_OK;
}

extern "C" int32_t b200vis_plan_row_order(uint32_t n, const uint32_t *parent, uint32_t *new_to_old) {
    if (n && (!parent || !new_to_old)) return B200VIS_ERR_INVALID_ARG;
    // children lists (ascending old row), then BFS per root in ascending root order
    std::vector<uint32_t> first(n + 1, 0), kids(n);
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t p = parent[r];
        if (p < n) first[p + 1]++;
        else if (p != kNoParent && p != kDetached) return B200VIS_ERR_PARENT_OUT_OF_RANGE;
    }
    for (uint32_t r = 0; r < n; ++r) first[r + 1] += first[r];
    { std::vector<uint32_t> cur(first.begin(), first.end() - 1);
      for (uint32_t r = 0; r < n; ++r) if (parent[r] < n) kids[cur[parent[r]]++] = r; }
    uint32_t out = 0;
    for (uint32_t r = 0; r < n; ++r) {
        if (parent[r] < n) continue;               // roots, flat entities and detached subtrees start a block
        const uint32_t head = out;
        new_to_old[out++] = r;
        for (uint32_t i = head; i < out; ++i) {
            const uint32_t c = new_to_old[i];
            for (uint32_t k = first[c]; k < first[c + 1]; ++k) new_to_old[out++] = kids[k];
        }
    }
    return out == n ? B200VIS_OK : B200VIS_ERR_HIERARCHY_CYCLE;   // rows on a cycle are never reached
}

// ------------------------------------------------------------------------------------------
// uploads
// ------------------------------------------------------------------------------------------
static int32_t stage_in(b200vis_ctx *ctx, const void *src, size_t bytes, size_t offset) {
    if (offset + bytes > ctx->stage_bytes) return fail(ctx, B200VIS_ERR_CAPACITY, "staging buffer too small");
    CU(cudaMemcpyAsync(ctx->d_stage + offset, src, bytes, cudaMemcpyDefault, ctx->stream));   // host or device source (UVA)
    return B200VIS_OK;
}

extern "C" int32_t b200vis_upload_transforms(b200vis_ctx *ctx, uint32_t first, uint32_t count, const float *trs) {
    CHECK_CTX();
    if (count && !trs) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_transforms: null");
    int32_t rc = check_range(ctx, first, count, "upload_transforms"); if (rc) return rc;
    rc = stage_in(ctx, trs, (size_t)count * 40, 0); if (rc) return rc;
    launch_unpack_trs(ctx->stream, ctx->rows, first, count, reinterpret_cast<const float *>(ctx->d_stage), 0);
    CU(cudaGetLastError());
    return B200VIS_OK;
}
extern "C" int32_t b200vis_upload_transforms_scattered(b200vis_ctx *ctx, uint32_t count, const uint32_t *rows, const float *trs) {
    CHECK_CTX();
    if (count && (!rows || !trs)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_transforms_scattered: null");
    if (count > ctx->cfg.max_entities) return fail(ctx, B200VIS_ERR_CAPACITY, "upload_transforms_scattered: count > max_entities");
    {   // sources already in device memory (a renderer / physics step on the same GPU): no staging copy
        cudaPointerAttributes pa{}, pb{};
        if (cudaPointerGetAttributes(&pa, rows) == cudaSuccess && cudaPointerGetAttributes(&pb, trs) == cudaSuccess) {
            if (pa.type == cudaMemoryTypeDevice && pb.type == cudaMemoryTypeDevice) {
                launch_scatter_trs(ctx->stream, ctx->rows, count, rows, trs);
                CU(cudaGetLastError());
                return B200VIS_OK;
            }
            // pinned (page-locked, mapped) host memory: the scatter kernel reads it over PCIe itself -- one launch instead
            // of two staging copies plus a launch.  The caller must not rewrite the buffers until the stream has passed.
            if (pa.type == cudaMemoryTypeHost && pb.type == cudaMemoryTypeHost && pa.devicePointer && pb.devicePointer) {
                launch_scatter_trs(ctx->stream, ctx->rows, count, static_cast<const uint32_t *>(pa.devicePointer),
                                   static_cast<const float *>(pb.devicePointer));
                CU(cudaGetLastError());
                return B200VIS_OK;
            }
        }
        cudaGetLastError();   // clear the error state cudaPointerGetAttributes leaves for unregistered host memory
    }
    const size_t off_rows = ((size_t)count * 40 + 15) & ~(size_t)15;
    int32_t rc = stage_in(ctx, trs, (size_t)count * 40, 0); if (rc) return rc;
    rc = stage_in(ctx, rows, (size_t)count * 4, off_rows); if (rc) return rc;
    launch_scatter_trs(ctx->stream, ctx->rows, count, reinterpret_cast<const uint32_t *>(ctx->d_stage + off_rows),
                       reinterpret_cast<const float *>(ctx->d_stage));
    CU(cudaGetLastError());
    return B200VIS_OK;
}
extern "C" int32_t b200vis_mark_transforms_changed(b200vis_ctx *ctx, uint32_t first, uint32_t count) {
    CHECK_CTX();
    int32_t rc = check_range(ctx, first, count, "mark_transforms_changed"); if (rc) return rc;
    launch_unpack_trs(ctx->stream, ctx->rows, first, count, nullptr, 1);
    CU(cudaGetLastError());
    return B200VIS_OK;
}
extern "C" int32_t b200vis_upload_global_transforms(b200vis_ctx *ctx, uint32_t first, uint32_t count, const float *gt) {
    CHECK_CTX();
    if (count && !gt) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_global_transforms: null");
    int32_t rc = check_range(ctx, first, count, "upload_global_transforms"); if (rc) return rc;
    rc = stage_in(ctx, gt, (size_t)count * 48, 0); if (rc) return rc;
    launch_unpack_gt(ctx->stream, ctx->rows, first, count, reinterpret_cast<const float *>(ctx->d_stage));
    CU(cudaGetLastError());
    return B200VIS_OK;
}
extern "C" int32_t b200vis_write_global_transforms_scattered(b200vis_ctx *ctx, uint32_t count, const uint32_t *rows, const float *gt) {
    CHECK_CTX();
    if (!ctx->topology_set) return fail(ctx, B200VIS_ERR_NOT_READY, "write_global_transforms_scattered: b200vis_set_topology has not been called");
    if (count && (!rows || !gt)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "write_global_transforms_scattered: null array");
    for (uint32_t i = 0; i < count; ++i)
        if (rows[i] >= ctx->n || row_is_dead(ctx, rows[i]))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "write_global_transforms_scattered: row %u (entry %u) out of range or despawned", rows[i], i);
    if (!count) return B200VIS_OK;
    // a row listed twice takes its last value: keep the last entry of every row, so that the scatter kernel's rows are distinct
    std::vector<uint64_t> key(count);
    for (uint32_t i = 0; i < count; ++i) key[i] = (uint64_t)rows[i] << 32 | i;
    std::sort(key.begin(), key.end());
    std::vector<uint32_t> urows; std::vector<float> ugt;
    urows.reserve(count); ugt.reserve((size_t)count * 12);
    for (uint32_t k = 0; k < count; ++k) {
        if (k + 1 < count && (key[k + 1] >> 32) == (key[k] >> 32)) continue;
        const uint32_t i = (uint32_t)key[k];
        urows.push_back(rows[i]);
        ugt.insert(ugt.end(), gt + (size_t)i * 12, gt + (size_t)i * 12 + 12);
    }
    const uint32_t m = (uint32_t)urows.size();
    const size_t off_rows = ((size_t)m * 48 + 15) & ~(size_t)15;
    int32_t rc = stage_in(ctx, ugt.data(), (size_t)m * 48, 0); if (rc) return rc;
    rc = stage_in(ctx, urows.data(), (size_t)m * 4, off_rows); if (rc) return rc;
    launch_write_gt_scattered(ctx->stream, ctx->rows, m, reinterpret_cast<const uint32_t *>(ctx->d_stage + off_rows),
                              reinterpret_cast<const float *>(ctx->d_stage));
    CU(cudaGetLastError());
    ctx->gt_ext_pending = true;
    ctx->gt_aos_valid = false;     // the dense write-back's copy of the column no longer holds what the host holds
    return B200VIS_OK;
}
extern "C" int32_t b200vis_upload_bounds(b200vis_ctx *ctx, uint32_t first, uint32_t count, const float *bounds,
                                         const uint8_t *flags, const uint8_t *class_mask, const uint64_t *layer_mask,
                                         const uint32_t *range_mask) {
    CHECK_CTX();
    if (count && (!bounds || !flags || !class_mask)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_bounds: null");
    int32_t rc = check_range(ctx, first, count, "upload_bounds"); if (rc) return rc;
    const size_t ob = 0, of = (size_t)count * 24, oc = of + (((size_t)count + 15) & ~(size_t)15);
    rc = stage_in(ctx, bounds, (size_t)count * 24, ob); if (rc) return rc;
    rc = stage_in(ctx, flags, count, of); if (rc) return rc;
    rc = stage_in(ctx, class_mask, count, oc); if (rc) return rc;
    launch_unpack_bounds(ctx->stream, ctx->rows, first, count, reinterpret_cast<const float *>(ctx->d_stage + ob),
                         ctx->d_stage + of, ctx->d_stage + oc, ctx->d_cls);
    CU(cudaGetLastError());
    if (layer_mask) {
        CU(cudaMemcpyAsync(ctx->d_layers + first, layer_mask, (size_t)count * 8, cudaMemcpyHostToDevice, ctx->stream));
        if (!ctx->have_layers) {
            // rows never uploaded keep the default layer (RenderLayers::default() = layer 0)
            std::vector<uint64_t> ones(ctx->cfg.max_entities, 1ull);
            CU(cudaStreamSynchronize(ctx->stream));
            if (first) CU(cudaMemcpy(ctx->d_layers, ones.data(), (size_t)first * 8, cudaMemcpyHostToDevice));
            const size_t tail = ctx->cfg.max_entities - (first + count);
            if (tail) CU(cudaMemcpy(ctx->d_layers + first + count, ones.data(), tail * 8, cudaMemcpyHostToDevice));
            ctx->have_layers = true;
        }
    }
    if (range_mask) {
        CU(cudaMemcpyAsync(ctx->d_range + first, range_mask, (size_t)count * 4, cudaMemcpyHostToDevice, ctx->stream));
        ctx->have_range = true;
    }
    ctx->bounds_set = true;
    ctx->lights_tag_dirty = true;   // flags were rewritten: re-verify that every light row is a sphere-from-GT row
    return B200VIS_OK;
}
extern "C" int32_t b200vis_upload_render_layers_ext(b200vis_ctx *ctx, uint32_t first, uint32_t count, const uint64_t *blocks) {
    CHECK_CTX();
    if (count && !blocks) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_render_layers_ext: null");
    int32_t rc = check_range(ctx, first, count, "upload_render_layers_ext"); if (rc) return rc;
    if (!ctx->d_layers_ext) CU(dalloc(&ctx->d_layers_ext, (size_t)ctx->cfg.max_entities * 3));   // rows never uploaded: blocks empty
    CU(cudaMemcpyAsync(ctx->d_layers_ext + (size_t)first * 3, blocks, (size_t)count * 24, cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->have_layers) {   // the general cull path reads block 0 per row too: default layer for everybody until uploaded
        std::vector<uint64_t> ones(ctx->cfg.max_entities, 1ull);
        CU(cudaStreamSynchronize(ctx->stream));
        CU(cudaMemcpy(ctx->d_layers, ones.data(), ones.size() * 8, cudaMemcpyHostToDevice));
        ctx->have_layers = true;
    }
    ctx->have_layers_ext = true;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_view_render_layers_ext(b200vis_ctx *ctx, uint32_t view, const uint64_t blocks[3]) {
    if (!ctx || view >= std::max<uint32_t>(ctx->cfg.max_views, kMaxViews)) return B200VIS_ERR_INVALID_ARG;   // views 0..7 always
    for (int k = 0; k < 3; ++k) ctx->view_layers_ext[view][k] = blocks ? blocks[k] : 0ull;
    if (ctx->light_ext_on) ctx->consts_dirty = true;   // the cluster kernels read the views' blocks from the frame blob
    return B200VIS_OK;
}
extern "C" int32_t b200vis_upload_view_visibility(b200vis_ctx *ctx, uint32_t first, uint32_t count, const uint8_t *vv) {
    CHECK_CTX();
    if (count && !vv) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_view_visibility: null");
    int32_t rc = check_range(ctx, first, count, "upload_view_visibility"); if (rc) return rc;
    rc = stage_in(ctx, vv, count, 0); if (rc) return rc;
    launch_unpack_vv(ctx->stream, ctx->rows, first, count, ctx->d_stage);
    CU(cudaGetLastError());
    return B200VIS_OK;
}

// ------------------------------------------------------------------------------------------
// per-frame constants
// ------------------------------------------------------------------------------------------
extern "C" int32_t b200vis_set_views(b200vis_ctx *ctx, uint32_t n_views, const b200vis_view *views) {
    if (!ctx) return B200VIS_ERR_INVALID_ARG;
    if (n_views > ctx->cfg.max_views) return fail(ctx, B200VIS_ERR_CAPACITY, "set_views: %u > max_views %u", n_views, ctx->cfg.max_views);
    if (n_views && !views) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_views: null");
    FrameConsts &fc = ctx->consts;
    fc.n_views = n_views;
    for (uint32_t v = 0; v < n_views; ++v) {
        DevView &d = fc.views[v];
        memcpy(d.hs, views[v].half_spaces, sizeof d.hs);
        d.layer_mask = views[v].layer_mask; d.flags = views[v].flags; d.range_index = views[v].range_view_index;
    }
    ctx->consts_dirty = true;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_view_count(b200vis_ctx *ctx, uint32_t n_views) {
    if (!ctx) return B200VIS_ERR_INVALID_ARG;
    if (n_views > ctx->cfg.max_views) return fail(ctx, B200VIS_ERR_CAPACITY, "set_view_count: %u > max_views %u", n_views, ctx->cfg.max_views);
    ctx->consts.n_views = n_views;
    ctx->consts_dirty = true;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_update_camera(b200vis_ctx *ctx, uint32_t view, const b200vis_camera *cam,
                                         const b200vis_cluster_config *cfg, const b200vis_cluster_feedback *fb,
                                         b200vis_cluster_view *out) {
    if (!ctx) return B200VIS_ERR_INVALID_ARG;
    if (view >= ctx->cfg.max_views || !cam) return fail(ctx, B200VIS_ERR_INVALID_ARG, "update_camera: bad view %u", view);
    float cfv[16], hs[6][4];
    host::perspective_infinite_reverse_rh(cam->fov_y, cam->aspect, cam->near_z, cfv);
    host::compute_frustum(cfv, cam->global_transform, cam->far_z, hs);
    DevView &d = ctx->consts.views[view];
    memcpy(d.hs, hs, sizeof d.hs);
    d.layer_mask = cam->layer_mask; d.flags = cam->flags; d.range_index = cam->range_view_index;
    if (ctx->consts.n_views <= view) ctx->consts.n_views = view + 1;
    ctx->consts_dirty = true;
    if (cfg) {
        static thread_local std::vector<float> scratch(3 * 4097 * 4);
        b200vis_cluster_view cv;
        int32_t rc = host::cluster_view_setup(cfg, cam->global_transform, cfv, hs, cam->layer_mask, fb, scratch.data(), &cv);
        if (rc) return fail(ctx, rc, "update_camera: cluster grid of view %u exceeds %d clusters", view, kMaxClusters);
        rc = b200vis_set_cluster_view(ctx, view, &cv);
        if (rc) return rc;
        if (out) *out = cv;
    } else {
        ctx->consts.cviews[view].enabled = 0;
        if (out) memset(out, 0, sizeof *out);
    }
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_lights(b200vis_ctx *ctx, uint32_t n_lights, const uint32_t *light_row, const float *range,
                                      const uint64_t *layer_mask) {
    CHECK_CTX();
    if (n_lights > ctx->cfg.max_lights) return fail(ctx, B200VIS_ERR_CAPACITY, "set_lights: %u > max_lights %u", n_lights, ctx->cfg.max_lights);
    if (n_lights && (!light_row || !range)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_lights: null");
    for (uint32_t i = 0; i < n_lights; ++i)
        if (light_row[i] >= ctx->cfg.max_entities || row_is_dead(ctx, light_row[i]))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_lights: light %u row %u out of range or despawned", i, light_row[i]);
    CU(cudaMemcpyAsync(ctx->d_light_row, light_row, (size_t)n_lights * 4, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_light_range, range, (size_t)n_lights * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (layer_mask) CU(cudaMemcpyAsync(ctx->d_light_layers, layer_mask, (size_t)n_lights * 8, cudaMemcpyHostToDevice, ctx->stream));
    ctx->h_light_row.assign(light_row, light_row + n_lights); ctx->h_light_range.assign(range, range + n_lights);
    ctx->lights.n = n_lights; ctx->lights.row = ctx->d_light_row; ctx->lights.range = ctx->d_light_range;
    ctx->lights.layers = layer_mask ? ctx->d_light_layers : nullptr;
    ctx->lights_tag_dirty = true;
    if (ctx->light_ext_on) { ctx->light_ext_on = false; ctx->consts_dirty = true; }   // every light's blocks 1..3 are empty again
    {   // the light blocks: stale snapshots out, ranges and layer masks in (rare: the tail of the frame in flight is joined first)
        const int32_t jrc = join_all(ctx); if (jrc) return jrc;
        const uint32_t cap = ctx->cl.max_lights;
        std::vector<uint8_t> blk(ctx->lrec_bytes, 0);
        float *rg = reinterpret_cast<float *>(blk.data() + (size_t)cap * 16);
        uint64_t *ly = reinterpret_cast<uint64_t *>(blk.data() + (size_t)cap * 20);
        for (uint32_t i = 0; i < n_lights; ++i) { rg[i] = range[i]; ly[i] = layer_mask ? layer_mask[i] : 1ull; }
        CU(cudaStreamSynchronize(ctx->stream));
        for (int k = 0; k < 3; ++k) CU(cudaMemcpy(ctx->d_lrec + k * ctx->lrec_bytes, blk.data(), ctx->lrec_bytes, cudaMemcpyHostToDevice));
    }
    return B200VIS_OK;
}

// blocks[n][3] -> dev (allocated with `cap` entries on first use); returns whether any block is nonzero
static int32_t upload_layer_blocks(b200vis_ctx *ctx, uint64_t **dev, uint32_t cap, uint32_t n, const uint64_t *blocks, bool *any) {
    *any = false;
    for (size_t i = 0; blocks && i < (size_t)n * 3; ++i) *any = *any || blocks[i] != 0ull;
    if (!*any) return B200VIS_OK;
    CU(cudaStreamSynchronize(ctx->stream));     // no kernel of the context still reads the old blocks
    if (!*dev) CU(dalloc(dev, (size_t)std::max<uint32_t>(cap, 1) * 3));
    CU(cudaMemcpy(*dev, blocks, (size_t)n * 24, cudaMemcpyHostToDevice));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_light_render_layers_ext(b200vis_ctx *ctx, uint32_t n_lights, const uint64_t *blocks) {
    CHECK_CTX_JOIN();   // the frame in flight may still be reading the lights' blocks
    if (ctx->cfg.world_size > 1)
        return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_light_render_layers_ext: world_size > 1 (the light records carry block 0 only)");
    if (n_lights != ctx->lights.n)
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_light_render_layers_ext: %u lights, b200vis_set_lights gave %u", n_lights, ctx->lights.n);
    bool any = false;
    const int32_t rc = upload_layer_blocks(ctx, &ctx->d_light_layers_ext, ctx->cfg.max_lights, n_lights, blocks, &any); if (rc) return rc;
    if (any != ctx->light_ext_on) ctx->consts_dirty = true;   // the frame blob gains / drops the views' blocks
    ctx->light_ext_on = any;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_shadow_item_render_layers_ext(b200vis_ctx *ctx, uint32_t n_items, const uint64_t *blocks) {
    CHECK_CTX_JOIN();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_shadow_item_render_layers_ext: world_size > 1");
    if (n_items != ctx->shadow.n_lights)
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_item_render_layers_ext: %u items, %u installed", n_items, ctx->shadow.n_lights);
    if (ctx->d_shadow_layers_ext && ctx->shadow_ext_cap < n_items) {   // the item capacity grew since the array was made
        CU(cudaStreamSynchronize(ctx->stream));
        CU(cudaFree(ctx->d_shadow_layers_ext)); ctx->d_shadow_layers_ext = nullptr;
    }
    if (!ctx->d_shadow_layers_ext) ctx->shadow_ext_cap = ctx->shadow_cap_lights;
    bool any = false;
    const int32_t rc = upload_layer_blocks(ctx, &ctx->d_shadow_layers_ext, ctx->shadow_ext_cap, n_items, blocks, &any); if (rc) return rc;
    ctx->shadow_ext_on = any;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_cluster_view_dims(const b200vis_ctx *ctx, uint32_t view, uint32_t dims[3]) {
    if (!ctx || !dims || view >= ctx->cfg.max_views) return B200VIS_ERR_INVALID_ARG;
    const DevClusterView &d = ctx->consts.cviews[view];
    for (int i = 0; i < 3; ++i) dims[i] = d.enabled ? d.dims[i] : 0u;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_cluster_view(b200vis_ctx *ctx, uint32_t view, const b200vis_cluster_view *p) {
    if (!ctx) return B200VIS_ERR_INVALID_ARG;
    if (view >= ctx->cfg.max_views || !p) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_cluster_view: bad view %u", view);
    DevClusterView &d = ctx->consts.cviews[view];
    memset(&d, 0, sizeof d);
    ctx->tab_x[view].clear(); ctx->tab_y[view].clear(); ctx->tab_z[view].clear(); ctx->tab_thr[view].clear();
    d.enabled = p->enabled;
    if (p->enabled) {
        const uint64_t nc = (uint64_t)p->dims[0] * p->dims[1] * p->dims[2];
        if (nc == 0 || nc > kMaxClusters) return fail(ctx, B200VIS_ERR_CAPACITY, "set_cluster_view: %llu clusters (max %d)", (unsigned long long)nc, kMaxClusters);
        if (!p->x_planes || !p->y_planes || !p->z_planes) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_cluster_view: null plane table");
        for (int i = 0; i < 3; ++i) d.dims[i] = p->dims[i];
        d.is_ortho = p->is_orthographic; d.n_clusters = (uint32_t)nc;
        memcpy(d.vfw, p->view_from_world, sizeof d.vfw); memcpy(d.cfv, p->clip_from_view, sizeof d.cfv);
        memcpy(d.scale, p->view_from_world_scale, sizeof d.scale); d.scale_max = p->view_from_world_scale_max;
        memcpy(d.frustum, p->frustum, sizeof d.frustum); d.layer_mask = p->layer_mask;
        ctx->tab_x[view].assign(p->x_planes, p->x_planes + (size_t)(p->dims[0] + 1) * 4);
        ctx->tab_y[view].assign(p->y_planes, p->y_planes + (size_t)(p->dims[1] + 1) * 4);
        ctx->tab_z[view].assign(p->z_planes, p->z_planes + (size_t)(p->dims[2] + 1) * 4);
        // view_z_to_z_slice through exact thresholds found with the host's libm (host_view.cpp)
        ctx->tab_thr[view].assign(((size_t)p->dims[2] + 3) & ~(size_t)3, NAN);
        host::z_slice_thresholds(p->cluster_factors, p->dims[2], p->is_orthographic != 0, ctx->tab_thr[view].data());
    }
    ctx->consts_dirty = true;
    return B200VIS_OK;
}

// Packs the working copy into the next pinned ring slot and issues one async copy.
static int32_t flush_consts(b200vis_ctx *ctx) {
    if (!ctx->consts_dirty) return B200VIS_OK;
    const int slot = ctx->ring_next;
    ctx->ring_next = (slot + 1) % b200vis_ctx::kRing;
    CU(cudaEventSynchronize(ctx->ring_ev[slot]));   // the copy issued kRing frames ago has long finished
    uint8_t *h = ctx->h_ring[slot];
    size_t off = (sizeof(FrameConsts) + 15) & ~(size_t)15;   // bytes; tables are float4 aligned
    for (uint32_t v = 0; v < ctx->consts.n_views && v < ctx->cfg.max_views; ++v) {
        DevClusterView &d = ctx->consts.cviews[v];
        if (!d.enabled) continue;
        std::vector<float> *tabs[4] = {&ctx->tab_x[v], &ctx->tab_y[v], &ctx->tab_z[v], &ctx->tab_thr[v]};
        uint32_t *offs[4] = {&d.x_off, &d.y_off, &d.z_off, &d.thr_off};
        for (int k = 0; k < 4; ++k) {
            *offs[k] = (uint32_t)(off / 4);
            memcpy(h + off, tabs[k]->data(), tabs[k]->size() * 4);
            off += (tabs[k]->size() * 4 + 15) & ~(size_t)15;
        }
    }
    ctx->consts.view_ext_off = 0;
    if (ctx->light_ext_on) {   // the views' RenderLayers blocks 1..3, for the lights that have some (k_cluster_assign<true>)
        ctx->consts.view_ext_off = (uint32_t)(off / 4);
        memcpy(h + off, ctx->view_layers_ext, sizeof ctx->view_layers_ext);
        off += (sizeof ctx->view_layers_ext + 15) & ~(size_t)15;
    }
    memcpy(h, &ctx->consts, sizeof(FrameConsts));
    CU(cudaMemcpyAsync(ctx->d_blob, h, off, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaEventRecord(ctx->ring_ev[slot], ctx->stream));
    ctx->blob_used = off;
    ctx->consts_dirty = false;
    ctx->blob_flushed = ctx->d_blob;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_record_frame_constants(b200vis_ctx *ctx, uint32_t *slot) {
    CHECK_CTX();
    if (!slot) return fail(ctx, B200VIS_ERR_INVALID_ARG, "record_frame_constants: null");
    ctx->consts_dirty = true;
    const int32_t rc = flush_consts(ctx); if (rc) return rc;
    b200vis_ctx::Recorded r;
    r.host = ctx->consts; r.bytes = ctx->blob_used; r.dev = nullptr;
    CU(cudaMalloc(reinterpret_cast<void **>(&r.dev), r.bytes));
    CU(cudaMemcpyAsync(r.dev, ctx->d_blob, r.bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->recorded.push_back(r);
    *slot = (uint32_t)ctx->recorded.size() - 1;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_use_recorded_frame_constants(b200vis_ctx *ctx, int32_t slot) {
    if (!ctx) return B200VIS_ERR_INVALID_ARG;
    if (slot >= (int32_t)ctx->recorded.size()) return fail(ctx, B200VIS_ERR_INVALID_ARG, "use_recorded_frame_constants: bad slot %d", slot);
    ctx->replay_slot = slot < 0 ? -1 : slot;
    return B200VIS_OK;
}
static const FrameConsts &active_consts(const b200vis_ctx *ctx) {
    return ctx->replay_slot >= 0 ? ctx->recorded[ctx->replay_slot].host : ctx->consts;
}
// The cull pass's view table for views base .. base + 7 (group base / 8).  n_views counts the group's own views only: the
// kernels index on[] / planes[] by it (k_cull's lane-per-view store reads cvw.on[lane] for lane < n_views).
static CullViews make_cull_views(const FrameConsts &fc, uint32_t base = 0) {
    CullViews c;
    memset(&c, 0, sizeof c);
    c.n_views = std::min<uint32_t>(kMaxViews, fc.n_views - base);
    for (uint32_t i = 0; base + i < fc.n_views && i < (uint32_t)kMaxViews; ++i) {
        const DevView &d = fc.views[base + i];
        c.on[i] = (d.flags & 3u) | ((d.layer_mask & 1ull) ? 4u : 0u); c.range_index[i] = d.range_index; c.layers[i] = d.layer_mask;
        for (int k = 0; k < 5; ++k) c.planes[i][k] = d.hs[k];
    }
    return c;
}

extern "C" int32_t b200vis_set_profiling(b200vis_ctx *ctx, int32_t enabled) {
    CHECK_CTX();
    if (enabled && !ctx->prof_ev) {
        ctx->prof_ev = new cudaEvent_t[b200vis_ctx::kProfFrames][6]();
        for (int i = 0; i < b200vis_ctx::kProfFrames; ++i) for (cudaEvent_t &e : ctx->prof_ev[i]) CU(cudaEventCreate(&e));
    }
    ctx->profiling = enabled != 0;
    ctx->prof_count = 0;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_collect_stage_times_ms(b200vis_ctx *ctx, float *tile_ms, float *expand_ms, float *cluster_ms, uint32_t *frames) {
    CHECK_CTX();
    if (!ctx->prof_ev) return fail(ctx, B200VIS_ERR_NOT_READY, "profiling was never enabled");
    { const int32_t rc = join_side(ctx); if (rc) return rc; }
    CU(cudaStreamSynchronize(ctx->stream));
    double s[3] = {0, 0, 0};
    for (int i = 0; i < ctx->prof_count; ++i) {
        float t = 0;
        CU(cudaEventElapsedTime(&t, ctx->prof_ev[i][0], ctx->prof_ev[i][1])); s[0] += t;   // tile pass (main stream)
        CU(cudaEventElapsedTime(&t, ctx->prof_ev[i][5], ctx->prof_ev[i][3])); s[1] += t;   // visible-list expansion
        CU(cudaEventElapsedTime(&t, ctx->prof_ev[i][3], ctx->prof_ev[i][4])); s[2] += t;   // cluster kernels ...
        CU(cudaEventElapsedTime(&t, ctx->prof_ev[i][2], ctx->prof_ev[i][5])); s[2] += t;   // ... incl. assign + exchange when issued first
    }
    if (tile_ms) *tile_ms = (float)s[0];
    if (expand_ms) *expand_ms = (float)s[1];
    if (cluster_ms) *cluster_ms = (float)s[2];
    if (frames) *frames = (uint32_t)ctx->prof_count;
    ctx->prof_count = 0;
    return B200VIS_OK;
}

// ------------------------------------------------------------------------------------------
// multi-GPU exchange buffers
// ------------------------------------------------------------------------------------------
extern "C" int32_t b200vis_comm_unique_id(uint8_t id[B200VIS_COMM_ID_BYTES]) {
    if (!id) return B200VIS_ERR_INVALID_ARG;
    if (!g_nccl.load()) return fail(nullptr, B200VIS_ERR_UNSUPPORTED, "libnccl.so.2 could not be loaded: %s", dlerror());
    const int rc = g_nccl.GetUniqueId(id);
    if (rc) return fail(nullptr, B200VIS_ERR_CUDA, "ncclGetUniqueId: %s", g_nccl.GetErrorString(rc));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_comm_init(b200vis_ctx *ctx, const uint8_t id[B200VIS_COMM_ID_BYTES]) {
    CHECK_CTX_JOIN();
    if (!id) return fail(ctx, B200VIS_ERR_INVALID_ARG, "comm_init: null id");
    if (ctx->cl.world <= 1) return fail(ctx, B200VIS_ERR_INVALID_ARG, "comm_init: the context was created with world_size <= 1");
    if (!g_nccl.load()) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "libnccl.so.2 could not be loaded: %s", dlerror());
    NcclApi::Id uid; memcpy(uid.b, id, sizeof uid.b);
    const int rc = g_nccl.CommInitRank(&ctx->nccl_comm, (int)ctx->cl.world, uid, (int)ctx->cl.rank);
    if (rc) { ctx->nccl_comm = nullptr; return fail(ctx, B200VIS_ERR_CUDA, "ncclCommInitRank: %s", g_nccl.GetErrorString(rc)); }
    if (!ctx->d_gather) CU(dalloc(&ctx->d_gather, (size_t)ctx->cl.world * ctx->slab_bytes / 4));
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->cl.send = ctx->d_slab; ctx->cl.recv = ctx->d_gather;
    return B200VIS_OK;
}
// Peer-memory exchange: export allocates this rank's gathered buffer and returns its CUDA IPC handle; the host gathers the
// handles of all ranks by any means; import maps the other ranks' buffers.  From then on b200vis_run(B200VIS_STAGE_ALL)
// pushes the slab into every rank's buffer with plain NVLink stores (k_slab_push) instead of calling ncclAllGather.
extern "C" int32_t b200vis_p2p_export(b200vis_ctx *ctx, uint8_t handle[B200VIS_P2P_HANDLE_BYTES]) {
    CHECK_CTX_JOIN();
    static_assert(sizeof(cudaIpcMemHandle_t) == B200VIS_P2P_HANDLE_BYTES, "IPC handle size");
    if (!handle) return fail(ctx, B200VIS_ERR_INVALID_ARG, "p2p_export: null");
    if (ctx->cl.world <= 1 || ctx->cl.world > 8) return fail(ctx, B200VIS_ERR_INVALID_ARG, "p2p_export: world_size must be 2..8");
    if (!ctx->d_xbuf) {
        const size_t data_words = (size_t)2 * ctx->cl.world * ctx->slab_bytes / 4;
        ctx->xbuf_flag_offset = data_words;
        void *p = nullptr;   // plain cudaMalloc: the allocation must be exportable through cudaIpcGetMemHandle
        CU(cudaMalloc(&p, (data_words + 64) * 4));
        CU(cudaMemset(p, 0, (data_words + 64) * 4));
        ctx->d_xbuf = static_cast<uint32_t *>(p);
        CU(dalloc(&ctx->d_push_done, 1));
    }
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, ctx->d_xbuf));
    memcpy(handle, &h, sizeof h);
    return B200VIS_OK;
}
extern "C" int32_t b200vis_p2p_import(b200vis_ctx *ctx, const uint8_t *handles) {
    CHECK_CTX_JOIN();
    if (!handles) return fail(ctx, B200VIS_ERR_INVALID_ARG, "p2p_import: null");
    if (!ctx->d_xbuf) return fail(ctx, B200VIS_ERR_NOT_READY, "p2p_import: call b200vis_p2p_export first");
    for (uint32_t r = 0; r < ctx->cl.world; ++r) {
        if (r == ctx->cl.rank) { ctx->peer_map[r] = ctx->d_xbuf; continue; }
        if (ctx->peer_map[r]) continue;
        cudaIpcMemHandle_t h; memcpy(&h, handles + (size_t)r * B200VIS_P2P_HANDLE_BYTES, sizeof h);
        void *p = nullptr;
        const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { cudaGetLastError(); return fail(ctx, B200VIS_ERR_UNSUPPORTED, "p2p_import: cudaIpcOpenMemHandle(rank %u): %s", r, cudaGetErrorString(e)); }
        ctx->peer_map[r] = p; ctx->peer_ipc[r] = true;
    }
    CU(cudaStreamSynchronize(ctx->stream));
    for (uint32_t r = 0; r < ctx->cl.world; ++r) {
        ctx->cl.peer[r] = static_cast<uint32_t *>(ctx->peer_map[r]);
        ctx->cl.peer_flags[r] = ctx->cl.peer[r] + ctx->xbuf_flag_offset;
    }
    ctx->cl.send = ctx->d_slab;
    ctx->p2p_ready = true;
    return B200VIS_OK;
}
// The same exchange for contexts that live in ONE process (a Bevy App is one process driving all its GPUs): no IPC handles,
// the contexts' gathered buffers are reached through plain peer access.  ctxs[r] must have been created with world_size = n and
// rank = r, each on its own device.  Afterwards the host thread simply calls b200vis_run(ctxs[r], B200VIS_STAGE_ALL) for every r
// (all launches are asynchronous; the list kernels wait for the peers' stamps on the device).
extern "C" int32_t b200vis_p2p_link(b200vis_ctx *const *ctxs, uint32_t n) {
    if (!ctxs || n < 2 || n > 8) return B200VIS_ERR_INVALID_ARG;
    for (uint32_t r = 0; r < n; ++r) {
        b200vis_ctx *ctx = ctxs[r];
        if (!ctx || ctx->cl.world != n || ctx->cl.rank != r)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "p2p_link: context %u must be created with world_size %u and rank %u", r, n, r);
        uint8_t unused[B200VIS_P2P_HANDLE_BYTES];
        const int32_t rc = b200vis_p2p_export(ctx, unused);      // allocates the gathered buffer + flags
        if (rc) return rc;
    }
    for (uint32_t r = 0; r < n; ++r) {
        b200vis_ctx *ctx = ctxs[r];
        CU(cudaSetDevice(ctx->device));
        for (uint32_t q = 0; q < n; ++q) {
            if (q != r && ctxs[q]->device != ctx->device) {
                int can = 0;
                CU(cudaDeviceCanAccessPeer(&can, ctx->device, ctxs[q]->device));
                if (!can) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "p2p_link: device %d cannot access device %d", ctx->device, ctxs[q]->device);
                const cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[q]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return fail(ctx, B200VIS_ERR_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e)); }
                cudaGetLastError();
            }
            ctx->peer_map[q] = ctxs[q]->d_xbuf; ctx->peer_ipc[q] = false;
            ctx->cl.peer[q] = ctxs[q]->d_xbuf;
            ctx->cl.peer_flags[q] = ctxs[q]->d_xbuf + ctxs[q]->xbuf_flag_offset;
        }
        CU(cudaStreamSynchronize(ctx->stream));
        ctx->cl.send = ctx->d_slab;
        ctx->p2p_ready = true;
    }
    return B200VIS_OK;
}
extern "C" int32_t b200vis_cluster_exchange_bytes(const b200vis_ctx *ctx, size_t *slab_bytes) {
    if (!ctx || !slab_bytes) return B200VIS_ERR_INVALID_ARG;
    *slab_bytes = ctx->slab_bytes;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_cluster_exchange_buffers(b200vis_ctx *ctx, void *send, void *recv) {
    CHECK_CTX_JOIN();
    if ((send == nullptr) != (recv == nullptr)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "exchange buffers: both or neither");
    CU(cudaStreamSynchronize(ctx->stream));
    if (send) {
        ctx->cl.send = static_cast<uint32_t *>(send); ctx->cl.recv = static_cast<const uint32_t *>(recv);
        CU(cudaMemsetAsync(send, 0, ctx->slab_bytes, ctx->stream));
    } else { ctx->cl.send = ctx->d_slab; ctx->cl.recv = ctx->d_slab; }
    ctx->ext_send = send; ctx->ext_recv = recv;
    return B200VIS_OK;
}

// ------------------------------------------------------------------------------------------
// run
// ------------------------------------------------------------------------------------------
// Makes the main stream wait for whatever the side stream still has in flight (cheap, asynchronous).
static int32_t join_side(b200vis_ctx *ctx) {
    if (ctx->tail_open) {   // work of an unfinished tail is on the side stream too
        CU(cudaEventRecord(ctx->ev_tile, ctx->side_stream));
        CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_tile, 0));
    }
    if (ctx->side_pending) {
        for (cudaEvent_t e : ctx->ev_side) CU(cudaStreamWaitEvent(ctx->stream, e, 0));
        ctx->side_pending = false;
    }
    return B200VIS_OK;
}
// additionally waits for an in-flight publish of the visible rows (readers of the sink / of the lists call this)
static int32_t join_all(b200vis_ctx *ctx) {
    if (ctx->pub_pending) { CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_pub, 0)); ctx->pub_pending = false; }
    return join_side(ctx);
}
extern "C" int32_t b200vis_tail_stream(b200vis_ctx *ctx, void **cuda_stream) {
    if (!ctx || !cuda_stream) return B200VIS_ERR_INVALID_ARG;
    *cuda_stream = ctx->pipeline ? static_cast<void *>(ctx->side_stream) : static_cast<void *>(ctx->stream);
    return B200VIS_OK;
}
extern "C" int32_t b200vis_join(b200vis_ctx *ctx) {
    CHECK_CTX();
    return join_all(ctx);
}

// b200vis_set_view_diff_sink, once per run that culls: the run's view -> slot map (views at or past the frame's view count
// have no slot; slotted = one past the last view with a slot), and the slots no view of the run names emptied on the tail
// stream ahead of the diff.  Only the slots that may hold entries are cleared, so a steady frame clears nothing; an
// inactive view's slot is emptied by k_view_diff.
static int32_t view_diff_slots_of_run(b200vis_ctx *ctx, cudaStream_t tail, uint32_t n_views, ViewSlots &vs, uint32_t &slotted) {
    std::fill(std::begin(vs.slot), std::end(vs.slot), kNoDiffSlot);
    slotted = 0;
    std::vector<uint8_t> named(ctx->vdiff_max_slots, 0);
    for (uint32_t v = 0; v < n_views && v < ctx->h_vdiff_slot.size(); ++v) {
        const uint32_t s = ctx->h_vdiff_slot[v];
        if (s == kNoDiffSlot) continue;
        vs.slot[v] = s; named[s] = 1; slotted = v + 1;
    }
    const size_t ws = ctx->vis.words_stride, cs = ctx->vis.chunks_stride;
    for (uint32_t s = 0; s < ctx->vdiff_max_slots; ++s) {
        if (ctx->vdiff_held[s] && !named[s]) {
            CU(cudaMemsetAsync(ctx->vdiff.prev + (size_t)s * 8 * ws, 0, 8 * ws * 4, tail));
            CU(cudaMemsetAsync(ctx->vdiff.prev_count + (size_t)s * cs, 0, cs * 4, tail));
        }
        ctx->vdiff_held[s] = named[s];
    }
    return B200VIS_OK;
}

// B200VIS_SWEEP_ORDER=fixed (experiment switch, read once per process): every sweep walks the rows in ascending order
static bool sweep_order_fixed() {
    static int v = -1;
    if (v < 0) { const char *e = getenv("B200VIS_SWEEP_ORDER"); v = (e && e[0] == 'f') ? 1 : 0; }
    return v != 0;
}
// Direction of the context's next full-world sweep: 0 ascending rows, 1 descending, alternating from sweep to sweep.  L2 holds
// about the last 40 MB a sweep touched; a sweep in the same direction reaches those rows last, after they have been evicted.
static uint32_t next_sweep_reversed(b200vis_ctx *ctx) {
    const uint32_t rev = ctx->sweep_count++ & 1u;
    return sweep_order_fixed() ? 0u : rev;
}

extern "C" int32_t b200vis_run(b200vis_ctx *ctx, uint32_t stages) {
    CHECK_CTX();
    if (!ctx->topology_set) return fail(ctx, B200VIS_ERR_NOT_READY, "run: b200vis_set_topology has not been called");
    if ((stages & B200VIS_STAGE_CULL) && !ctx->bounds_set) return fail(ctx, B200VIS_ERR_NOT_READY, "run: bounds/flags were never uploaded");
    cudaStream_t st = ctx->stream;
    const bool do_prop = stages & B200VIS_STAGE_PROPAGATE, do_cull = stages & B200VIS_STAGE_CULL;
    const bool has_assign = stages & B200VIS_STAGE_CLUSTER_ASSIGN, has_lists = stages & B200VIS_STAGE_CLUSTER_LISTS;
    // pending external GlobalTransform writes: only kernel 1b has the marked instantiation
    const bool gt_ext = do_prop && ctx->gt_ext_pending;
    if (gt_ext && !tile_kernel_is_default()) {
        const char *e = getenv("B200VIS_TILE_KERNEL");
        return fail(ctx, B200VIS_ERR_UNSUPPORTED, "run: GlobalTransforms written by b200vis_write_global_transforms_scattered are pending, "
                    "and B200VIS_TILE_KERNEL=%s selects a tile kernel that does not read them (unset it, or set it to tma)", e ? e : "");
    }
    // ---- continuation of an open tail: CLUSTER_LISTS after the host's all-gather, still on the side stream --------
    if (ctx->pipeline && ctx->tail_open && stages == B200VIS_STAGE_CLUSTER_LISTS) {
        ClusterBufs cl = ctx->cl;
        cl.blob = reinterpret_cast<const float *>(ctx->open_fc);
        cudaStream_t tail = ctx->side_stream;
        launch_cluster_lists(tail, ctx->open_fc, cl, ctx->d_stats, ctx->cfg.max_views);
        if (ctx->have_sink)
            launch_publish_clusters(tail, ctx->open_fc, cl, ctx->sink_off_d, ctx->sink_idx_d, ctx->sink.cluster_capacity, ctx->d_stats,
                                    ctx->sink_stats_d, ctx->open_frame % 3u, ctx->open_frame + 1u, ctx->cfg.max_views,
                                    ctx->view_stats_d);
        CU(cudaEventRecord(ctx->ev_side[ctx->open_frame % 3u], tail));
        ctx->side_pending = true; ctx->tail_open = false;
        CU(cudaGetLastError());
        return B200VIS_OK;
    }
    // Pipelined mode: a whole frame (or a frame up to the cluster exchange).  The tail of frame f (expand + cluster) goes to
    // the side stream and overlaps the tile passes of frames f+1 AND f+2: frame f+2's tile pass only waits for frame f's
    // list EXPANSION (it reuses frame f's visible masks and counters, two / three copies), frame f+3's for frame f's whole
    // tail (frame constants and light snapshots: three copies).  So a tail may take up to two frame periods -- which is what
    // the multi-GPU case needs, where the tail contains the cluster exchange and waits on other GPUs.
    const bool pipelined = ctx->pipeline && do_prop && do_cull && has_assign && !ctx->tail_open;
    const uint32_t frame = ctx->frame;
    const uint32_t cslot = frame % 3u, mslot = frame & 1u;
    if (pipelined) {
        if (ctx->side_pending && frame >= 2) CU(cudaStreamWaitEvent(st, ctx->ev_expand[mslot], 0));   // expansion of frame f-2
        if (ctx->side_pending && frame >= 3) CU(cudaStreamWaitEvent(st, ctx->ev_side[cslot], 0));     // tail of frame f-3
    } else {
        if (ctx->tail_open) {   // an abandoned open tail: close it so that the event chain stays consistent
            CU(cudaEventRecord(ctx->ev_side[ctx->open_frame % 3u], ctx->side_stream));
            ctx->side_pending = true; ctx->tail_open = false;
        }
        const int32_t rc = join_side(ctx); if (rc) return rc;
    }
    ClusterBufs cl = ctx->cl;
    const FrameConsts *fc;
    if (ctx->replay_slot >= 0) {   // constants already resident in HBM (recorded earlier): no host work, no copy
        fc = reinterpret_cast<const FrameConsts *>(ctx->recorded[ctx->replay_slot].dev);
    } else {
        ctx->d_blob = ctx->d_blob2[cslot];          // the side stream may still read the other two copies
        ctx->d_consts = reinterpret_cast<FrameConsts *>(ctx->d_blob);
        // each copy must be current: a pipelined frame rewrites its slot, and so does any run whose slot is not the one last
        // flushed (CULL advances the frame, so a CLUSTER run right behind it reads the next slot)
        ctx->consts_dirty = ctx->consts_dirty || pipelined || ctx->blob_flushed != ctx->d_blob;
        const int32_t rc = flush_consts(ctx); if (rc) return rc;
        fc = ctx->d_consts;
    }
    cl.blob = reinterpret_cast<const float *>(fc);
    const FrameConsts &afc = active_consts(ctx);
    CullViews cvw = make_cull_views(afc);
    Rows R = ctx->rows;
    R.layers = ctx->have_layers ? ctx->d_layers : nullptr;
    R.layers_ext = ctx->have_layers_ext ? ctx->d_layers_ext : nullptr;
    if (ctx->have_layers_ext) memcpy(cvw.layers_ext, ctx->view_layers_ext, sizeof cvw.layers_ext);
    R.range = ctx->have_range ? ctx->d_range : nullptr;
    R.range_se = ctx->d_range_se; R.range_use_aabb = ctx->d_range_ua;
    R.range_views = ctx->d_range_views; R.n_range_views = ctx->n_range_views;
    R.rank = ctx->rank_identity ? nullptr : ctx->d_rank;
    R.row_of_rank = ctx->rank_identity ? nullptr : ctx->d_row_of_rank;
    VisibleBufs vb = ctx->vis;
    vb.mask = ctx->vis.mask + (size_t)mslot * ctx->vis.words_stride * ctx->cfg.max_views;
    const uint32_t n_pass = ctx->pass_begin.empty() ? 0 : (uint32_t)ctx->pass_begin.size() - 1;
    // views past the eighth: group passes of k_cull behind the frame's last tile pass (see launch_cull_group)
    const bool view_groups = do_cull && n_pass && afc.n_views > (uint32_t)kMaxViews;
    R.dirty = nullptr;
    R.light_snap = nullptr; R.light_ord = nullptr; R.n_lights = 0;
    if (do_prop && ctx->static_opt && n_pass > 1) {
        CU(cudaMemsetAsync(ctx->d_dirty, 0, ctx->n, st));
        R.dirty = ctx->d_dirty;
        launch_mark_dirty_global(st, R);
    }
    // Light snapshot by the tile kernel itself: needs every light row tagged with its ordinal (one-off, on change).
    bool tile_snap = false;
    if (pipelined && ctx->lights.n) {
        if (ctx->lights_tag_dirty) {
            const uint32_t one = 1;
            CU(cudaMemcpyAsync(ctx->d_tag_flag, &one, 4, cudaMemcpyHostToDevice, st));
            // rows that were lights under the previous list lose their ordinal: the whole column is rewritten
            CU(cudaMemsetAsync(ctx->d_light_ord, 0xFF, std::max<size_t>(ctx->cfg.max_entities, 1) * 4, st));
            launch_tag_lights(st, R, ctx->lights, ctx->d_light_ord, ctx->d_tag_flag);
            uint32_t ok = 0;
            CU(cudaMemcpyAsync(&ok, ctx->d_tag_flag, 4, cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            ctx->lights_tagged = ok != 0; ctx->lights_tag_dirty = false;
        }
        bool any_small = false;
        for (uint32_t x : ctx->pass_small) any_small |= x != 0;
        tile_snap = ctx->lights_tagged && tile_kernel_publishes_light_snapshot() && !any_small;   // the 32-thread kernel does not publish snapshots
        tile_snap = tile_snap && !view_groups;   // a light only a view >= 8 sees is visible after the group passes only
        if (tile_snap) {
            R.light_snap = ctx->light_snap_slot(cslot);
            R.light_ord = ctx->d_light_ord; R.n_lights = ctx->lights.n;
        }
    }
    cudaEvent_t *pe = (ctx->profiling && ctx->prof_count < b200vis_ctx::kProfFrames) ? ctx->prof_ev[ctx->prof_count++] : nullptr;
    if (pe) CU(cudaEventRecord(pe[0], st));
    if (do_prop || do_cull) {
        const uint32_t tile_stages = (do_prop ? 1u : 0u) | (do_cull ? 2u : 0u);
        if (do_prop) {
            for (uint32_t p = 0; p < n_pass && gt_ext; ++p) {
                // the whole pass, small tiles (B200VIS_SPLIT_DEEP_TILES) included, through kernel 1b's marked instantiation
                const uint32_t b = ctx->pass_begin[p];
                launch_propagate_cull_ext(st, R, ctx->d_tiles + b, ctx->pass_begin[p + 1] - b, cvw, vb, ctx->d_stats, tile_stages,
                                          (uint32_t)ctx->static_opt, cslot, ctx->d_tile_ticket, &ctx->tile_ticket_base,
                                          next_sweep_reversed(ctx));
            }
            if (gt_ext) ctx->gt_ext_pending = false;
            for (uint32_t p = 0; p < n_pass && !gt_ext; ++p) {
                const uint32_t ns = p < ctx->pass_small.size() ? ctx->pass_small[p] : 0u, b = ctx->pass_begin[p];
                if (ns) launch_propagate_cull_small(st, R, ctx->d_tiles + b, ns, cvw, vb, ctx->d_stats, tile_stages, (uint32_t)ctx->static_opt, cslot);
                if (tile_kernel_is_warp())
                    launch_tile_warp(st, R, ctx->d_wtiles + b + ns, ctx->d_sched, ctx->pass_begin[p + 1] - b - ns,
                                     cvw, vb, ctx->d_stats, tile_stages, (uint32_t)ctx->static_opt, cslot, ctx->d_tile_counter);
                else
                    launch_propagate_cull(st, R, ctx->d_tiles + b + ns, ctx->pass_begin[p + 1] - b - ns,
                                          cvw, vb, ctx->d_stats, tile_stages, (uint32_t)ctx->static_opt, cslot, ctx->d_tile_ticket, &ctx->tile_ticket_base,
                                          p < ctx->pass_named.size() && ctx->pass_named[p] != 0, next_sweep_reversed(ctx),
                                          ctx->gt_stage_full ? nullptr : ctx->d_tile_hint + b + ns);
            }
        } else if (n_pass) {
            launch_cull(st, R, cvw, vb, ctx->d_stats, cslot, next_sweep_reversed(ctx));
        }
        for (uint32_t b = kMaxViews; view_groups && b < afc.n_views; b += kMaxViews) {
            CullViews g = make_cull_views(afc, b);
            if (ctx->have_layers_ext) memcpy(g.layers_ext, ctx->view_layers_ext[b], sizeof g.layers_ext);
            launch_cull_group(st, R, g, vb, ctx->d_stats, cslot, b, next_sweep_reversed(ctx));
        }
    }
    Lights lights = ctx->lights;
    lights.snap = nullptr;
    // lights with RenderLayers blocks 1..3: only with the views' blocks in this frame's constants (a frame recorded before the
    // light blocks were set has none, and its views then see block 0 alone)
    lights.layers_ext = ctx->light_ext_on && afc.view_ext_off ? ctx->d_light_layers_ext : nullptr;
    cudaStream_t tail = st;
    if (pipelined) {
        lights.snap = ctx->light_snap_slot(cslot);
        if (!tile_snap) launch_snapshot_lights(st, R, lights, const_cast<float4 *>(lights.snap));
        if (pe) CU(cudaEventRecord(pe[1], st));
        CU(cudaEventRecord(ctx->ev_tile, st));
        tail = ctx->side_stream;
        CU(cudaStreamWaitEvent(tail, ctx->ev_tile, 0));
    } else if (pe) CU(cudaEventRecord(pe[1], st));
    if (pe) CU(cudaEventRecord(pe[2], tail));
    // Multi-GPU: the cluster exchange is the one step of the tail that waits on other GPUs, so it goes FIRST -- assign and
    // the slab push / all-gather are issued before the visible-list expansion (they do not depend on it), and the peers'
    // data travels while this rank expands its lists.
    const bool exchange_first = has_assign && has_lists && cl.world > 1;
    // Several GPUs, built-in collective: what travels is the LIGHT RECORD block (28 bytes per light: position + ViewVisibility
    // from this frame's tile pass, range, layers) instead of the cluster x light bit slabs, and every rank then runs the
    // one-launch cluster stage over all ranks' lights -- the same kernel, the same ordinals (rank * capacity + local), the same
    // Clusters feedback on every rank, and a few KB on the wire instead of V x words x 16 KB.  Used whenever the gathered bit
    // matrix fits the fused kernel's distributed shared memory (<= 6400 lights in all); B200VIS_EXCHANGE_WHAT=slabs (or a host-
    // driven / peer-store exchange) keeps the slab path.
    static int records_env = -1;
    if (records_env < 0) { const char *e = getenv("B200VIS_EXCHANGE_WHAT"); records_env = (e && e[0] == 's') ? 0 : 1; }
    const bool records = exchange_first && records_env && (ctx->nccl_comm || ctx->p2p_ready) && ctx->ext_send == nullptr &&
                         cluster_fused_fits(cl.world * cl.max_lights);
    bool fused_clusters = false;     // both cluster stages in this call and all lights at hand: one launch does assign + lists
    // Pipelined frames: the cluster branch of the tail (exchange -> cluster kernel(s) -> bindings) depends on the tile pass only,
    // not on the list expansion, and its first step may wait for other GPUs: it gets a stream of its own (`ctail`) beside the
    // expansion / visible-list publish on `tail`; the two meet again before the stats + cluster lists are published.  The
    // branch also waits for the previous frame's tail (its cluster lists and stats are single-buffered).
    static int branch_env = -1;
    if (branch_env < 0) { const char *e = getenv("B200VIS_CLUSTER_BRANCH"); branch_env = (e && e[0] == '0') ? 0 : 1; }
    const bool branch = pipelined && has_assign && has_lists && branch_env && ctx->clus_stream != nullptr;
    cudaStream_t ctail = tail;
    if (branch) {
        ctail = ctx->clus_stream;
        CU(cudaStreamWaitEvent(ctail, ctx->ev_tile, 0));
        if (ctx->side_pending && frame >= 1) CU(cudaStreamWaitEvent(ctail, ctx->ev_side[(frame + 2u) % 3u], 0));
    }
    auto issue_assign_and_exchange = [&]() -> int32_t {
        if (records) {
            if (!(pipelined && ctx->lights.n)) {      // no snapshot was taken with the tile pass: take it now (same stream order)
                Lights lsnap = ctx->lights;
                launch_snapshot_lights(ctail, R, lsnap, ctx->light_snap_slot(cslot));
            }
            if (ctx->p2p_ready) {        // peer stores over NVLink + stamps; the cluster kernel waits for every rank's stamp
                cl.p2p = 1; cl.xparity = mslot; cl.stamp = frame + 1u;
                launch_record_push(ctail, reinterpret_cast<const uint32_t *>(ctx->d_lrec + (size_t)cslot * ctx->lrec_bytes), (uint32_t)(ctx->lrec_bytes / 4), cl);
                return B200VIS_OK;
            }
            const int nrc = g_nccl.AllGather(ctx->d_lrec + (size_t)cslot * ctx->lrec_bytes, ctx->d_lrec_all, ctx->lrec_bytes / 4, kNcclUint32,
                                             ctx->nccl_comm, ctail);
            if (nrc) return fail(ctx, B200VIS_ERR_CUDA, "ncclAllGather: %s", g_nccl.GetErrorString(nrc));
            return B200VIS_OK;
        }
        if (has_assign && has_lists && cl.world == 1 && ctx->ext_send == nullptr && lights.n)
            fused_clusters = launch_cluster_fused(ctail, R, lights, fc, cl, ctx->d_stats, ctx->cfg.max_views);
        if ((stages & B200VIS_STAGE_CLUSTER_ASSIGN) && !fused_clusters)
            launch_cluster_assign(ctail, R, lights, fc, cl, ctx->d_stats, ctx->cfg.max_views);
        if (has_assign && has_lists && cl.world > 1) {
            if (ctx->p2p_ready) {
                // peer stores over NVLink + stamps; k_cluster_lists waits for every rank's stamp of this frame
                cl.p2p = 1; cl.xparity = mslot; cl.stamp = frame + 1u;
                cl.recv = ctx->d_xbuf + (size_t)mslot * cl.world * (ctx->slab_bytes / 4);
                launch_slab_push(ctail, fc, cl, ctx->d_push_done, ctx->cfg.max_views);
            } else {
                // the ONE data-path collective: rank-major all-gather of the fixed-size cluster x light slabs over NVLink
                if (!ctx->nccl_comm) return fail(ctx, B200VIS_ERR_NOT_READY, "run(ALL) with world_size > 1 needs b200vis_p2p_import or b200vis_comm_init (or run ASSIGN and LISTS separately around your own all-gather)");
                const int nrc = g_nccl.AllGather(cl.send, const_cast<uint32_t *>(cl.recv), ctx->slab_bytes / 4, kNcclUint32, ctx->nccl_comm, ctail);
                if (nrc) return fail(ctx, B200VIS_ERR_CUDA, "ncclAllGather: %s", g_nccl.GetErrorString(nrc));
            }
        }
        return B200VIS_OK;
    };
    if (exchange_first) { const int32_t rc = issue_assign_and_exchange(); if (rc) return rc; }
    if (pe) CU(cudaEventRecord(pe[5], tail));
    if (do_cull && ctx->pub_pending) { CU(cudaStreamWaitEvent(tail, ctx->ev_pub, 0)); ctx->pub_pending = false; }   // lists are rewritten
    ViewDiff vd = ctx->vdiff;
    ViewSlots vs;
    uint32_t slotted = 0;
    if (do_cull && vd.added) {                   // ahead of the expansion, which consumes the masks
        const int32_t rc = view_diff_slots_of_run(ctx, tail, afc.n_views, vs, slotted); if (rc) return rc;
        vd.keys = ctx->d_keys;                   // a compaction swaps the key buffers
        launch_view_diff(tail, vb, vd, vs, R.row_of_rank, fc, cslot, slotted);
    }
    if (do_cull) {
        launch_expand_visible(tail, vb, ctx->diff_on ? ctx->diff : DiffBufs{}, R.row_of_rank, fc, ctx->d_stats, cslot, ctx->n, ctx->cfg.max_views);
        if (pipelined) CU(cudaEventRecord(ctx->ev_expand[mslot], tail));   // this frame's masks / counters are free again
        if (ctx->diff_on && ctx->diff_sink_rows_d)
            launch_publish_visible_diff(tail, vb, ctx->diff, ctx->diff_sink_rows_d, ctx->diff_sink_cap, ctx->diff_sink_counts_d,
                                        active_consts(ctx).n_views, ctx->cfg.max_views);
        if (ctx->ent_sink_d)
            launch_emit_visible_entities(tail, vb, R.rank, ctx->d_keys, fc, ctx->d_stats, ctx->n, ctx->cfg.max_views, ctx->d_ent_counts,
                                         ctx->ent_chunks, ctx->ent_sink_d, ctx->ent_cap, ctx->ent_off_d);
        if (vd.added) launch_emit_view_diff(tail, vb, vd, vs, afc.n_views, slotted);
    }
    if (do_cull && ctx->have_sink && ctx->sink_rows_d) {
        // posting ~1 MB of visible rows over PCIe takes tens of microseconds: in the serial (non-pipelined) case do it on the
        // side stream so it overlaps the cluster kernels; every later consumer joins the side stream
        cudaStream_t pub = tail;
        if (!pipelined) {
            CU(cudaEventRecord(ctx->ev_tile, tail));
            CU(cudaStreamWaitEvent(ctx->side_stream, ctx->ev_tile, 0));
            pub = ctx->side_stream;
        }
        launch_publish_visible(pub, vb, ctx->d_stats, ctx->sink_rows_d, ctx->sink.visible_capacity, ctx->n, active_consts(ctx).n_views, ctx->sink_cls_d);
        if (!pipelined) { CU(cudaEventRecord(ctx->ev_pub, pub)); ctx->pub_pending = true; }
    }
    if (pe) CU(cudaEventRecord(pe[3], tail));
    if (!exchange_first) { const int32_t rc = issue_assign_and_exchange(); if (rc) return rc; }
    if (records) {
        Lights lg{};
        lg.n = cl.world * cl.max_lights; lg.per_rank = cl.max_lights; lg.block_bytes = (uint32_t)ctx->lrec_bytes; lg.blocks = ctx->d_lrec_all;
        if (ctx->p2p_ready) {       // the gathered buffer the peers wrote into: one slab-sized region per (parity, rank), the block at its front
            lg.block_bytes = (uint32_t)ctx->slab_bytes;
            lg.blocks = reinterpret_cast<const uint8_t *>(ctx->d_xbuf + (size_t)mslot * cl.world * (ctx->slab_bytes / 4));
        }
        fused_clusters = launch_cluster_fused(ctail, R, lg, fc, cl, ctx->d_stats, ctx->cfg.max_views);
        if (!fused_clusters) return fail(ctx, B200VIS_ERR_CUDA, "run: the cluster kernel could not be launched over the gathered light records");
    }
    if ((stages & B200VIS_STAGE_CLUSTER_LISTS) && !fused_clusters)
        launch_cluster_lists(ctail, fc, cl, ctx->d_stats, ctx->cfg.max_views);
    if ((stages & B200VIS_STAGE_CLUSTER_LISTS) && ctx->bind.mode)
        launch_pack_cluster_bindings(ctail, fc, cl, ctx->bind, ctx->cfg.max_views);
    if (branch) { CU(cudaEventRecord(ctx->ev_clus, ctail)); CU(cudaStreamWaitEvent(tail, ctx->ev_clus, 0)); }   // the branches meet
    // (b200vis_step with clusters runs CLUSTER right behind PROPAGATE|CULL: that run publishes the stats block once for both)
    if (ctx->have_sink && (do_cull || (stages & B200VIS_STAGE_CLUSTER_LISTS)) && !(ctx->step_defers_stats && !(stages & B200VIS_STAGE_CLUSTER_LISTS)))
        launch_publish_clusters(tail, fc, cl, (stages & B200VIS_STAGE_CLUSTER_LISTS) ? ctx->sink_off_d : nullptr, ctx->sink_idx_d,
                                ctx->sink.cluster_capacity, ctx->d_stats, ctx->sink_stats_d, do_cull ? cslot : (frame + 2u) % 3u, frame + (do_cull ? 1u : 0u), ctx->cfg.max_views,
                                ctx->view_stats_d);
    if (pe) CU(cudaEventRecord(pe[4], tail));
    if (pipelined) {
        if (has_lists) { CU(cudaEventRecord(ctx->ev_side[cslot], tail)); ctx->side_pending = true; }
        else { ctx->tail_open = true; ctx->open_frame = frame; ctx->open_fc = fc; }
    }
    CU(cudaGetLastError());
    if (do_cull) { ctx->frame++; ctx->parity = ctx->frame % 3u; }
    return B200VIS_OK;
}

// ------------------------------------------------------------------------------------------
// downloads (synchronous: the host buffers are valid on return)
// ------------------------------------------------------------------------------------------
extern "C" int32_t b200vis_download_frame_stats(b200vis_ctx *ctx, b200vis_frame_stats *out) {
    CHECK_CTX_JOIN();
    if (!out) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_frame_stats: null");
    CU(cudaMemcpyAsync(ctx->h_stats, ctx->d_stats, sizeof(DevStats), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const DevStats &s = *ctx->h_stats;
    memset(out, 0, sizeof *out);
    for (int v = 0; v < kMaxViews; ++v) {
        out->visible_count[v] = s.visible_count[v];
        out->cluster_index_count[v] = s.cl_index_count[v];
        memcpy(&out->cluster_farthest_z[v], &s.cl_farthest_bits[v], 4);
        out->cluster_index_overflow[v] = s.cl_overflow[v];
    }
    const uint32_t lp = (ctx->frame + 2u) % 3u;   // slot the last CULL frame (frame - 1) accumulated into
    out->gt_changed_count = s.changed[lp][0]; out->vv_changed_count = s.changed[lp][1]; out->frame = ctx->frame;
    ctx->last_gt_changed = out->gt_changed_count;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_download_view_stats(b200vis_ctx *ctx, uint32_t first_view, uint32_t count, uint32_t *visible_count,
                                               uint32_t *cluster_index_count, float *cluster_farthest_z, uint32_t *cluster_index_overflow) {
    CHECK_CTX_JOIN();
    if ((uint64_t)first_view + count > ctx->cfg.max_views)
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_view_stats: views [%u, %u) exceed max_views %u", first_view, first_view + count,
                    ctx->cfg.max_views);
    CU(cudaMemcpyAsync(ctx->h_stats, ctx->d_stats, sizeof(DevStats), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const DevStats &s = *ctx->h_stats;
    for (uint32_t i = 0; i < count; ++i) {
        const uint32_t v = first_view + i;
        if (visible_count) visible_count[i] = s.visible_count[v];
        if (cluster_index_count) cluster_index_count[i] = s.cl_index_count[v];
        if (cluster_farthest_z) memcpy(&cluster_farthest_z[i], &s.cl_farthest_bits[v], 4);
        if (cluster_index_overflow) cluster_index_overflow[i] = s.cl_overflow[v];
    }
    return B200VIS_OK;
}

extern "C" int32_t b200vis_download_global_transforms(b200vis_ctx *ctx, uint32_t first, uint32_t count, float *gt,
                                                      uint32_t stride, uint8_t *changed) {
    CHECK_CTX_JOIN();
    int32_t rc = check_range(ctx, first, count, "download_global_transforms"); if (rc) return rc;
    if (gt && stride != 12 && stride != 16) return fail(ctx, B200VIS_ERR_INVALID_ARG, "stride_floats must be 12 or 16");
    cudaStream_t st = ctx->stream;
    if (gt) {
        launch_pack_gt(st, ctx->rows, first, count, reinterpret_cast<float *>(ctx->d_stage), stride);
        CU(cudaMemcpyAsync(gt, ctx->d_stage, (size_t)count * stride * 4, cudaMemcpyDeviceToHost, st));
    }
    if (changed) {
        CU(cudaStreamSynchronize(st));
        launch_pack_state(st, ctx->rows, first, count, ctx->d_stage, S_GT_CHANGED);
        CU(cudaMemcpyAsync(changed, ctx->d_stage + count, count, cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_view_visibility(b200vis_ctx *ctx, uint32_t first, uint32_t count, uint8_t *vv, uint8_t *changed) {
    CHECK_CTX_JOIN();
    int32_t rc = check_range(ctx, first, count, "download_view_visibility"); if (rc) return rc;
    cudaStream_t st = ctx->stream;
    launch_pack_state(st, ctx->rows, first, count, ctx->d_stage, S_VV_CHANGED);
    if (vv) CU(cudaMemcpyAsync(vv, ctx->d_stage, count, cudaMemcpyDeviceToHost, st));
    if (changed) CU(cudaMemcpyAsync(changed, ctx->d_stage + count, count, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_visible(b200vis_ctx *ctx, uint32_t view, uint32_t *rows, uint32_t capacity, uint32_t *count) {
    CHECK_CTX_JOIN();
    if (view >= ctx->cfg.max_views || !count) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_visible: bad argument");
    cudaStream_t st = ctx->stream;
    CU(cudaMemcpyAsync(ctx->h_stats, ctx->d_stats, sizeof(DevStats), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t c = ctx->h_stats->visible_count[view];   // an inactive view keeps its last list (mod.rs:780-782)
    *count = c;
    if (rows) {
        if (c > capacity) return fail(ctx, B200VIS_ERR_CAPACITY, "download_visible: %u rows > capacity %u", c, capacity);
        CU(cudaMemcpyAsync(rows, ctx->vis.lists + (size_t)view * ctx->vis.list_stride, (size_t)c * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_visible_classes(b200vis_ctx *ctx, uint32_t view, uint8_t *classes, uint32_t capacity, uint32_t *count) {
    CHECK_CTX_JOIN();
    if (view >= ctx->cfg.max_views || !count) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_visible_classes: bad argument");
    cudaStream_t st = ctx->stream;
    CU(cudaMemcpyAsync(ctx->h_stats, ctx->d_stats, sizeof(DevStats), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t c = ctx->h_stats->visible_count[view];
    *count = c;
    if (classes) {
        if (c > capacity) return fail(ctx, B200VIS_ERR_CAPACITY, "download_visible_classes: %u entries > capacity %u", c, capacity);
        CU(cudaMemcpyAsync(classes, ctx->vis.classes + (size_t)view * ctx->vis.list_stride, c, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_clusters(b200vis_ctx *ctx, uint32_t view, uint32_t *offsets, uint32_t *indices,
                                             uint32_t indices_capacity, uint32_t *total) {
    CHECK_CTX_JOIN();
    if (view >= ctx->cfg.max_views || !offsets || !total) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_clusters: bad argument");
    const DevClusterView &cv = active_consts(ctx).cviews[view];
    const uint32_t nc = cv.enabled ? cv.n_clusters : 0;
    cudaStream_t st = ctx->stream;
    CU(cudaMemcpyAsync(offsets, ctx->cl.offsets + (size_t)view * (kMaxClusters + 1), (size_t)(nc + 1) * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    *total = offsets[nc];
    if (*total > ctx->cl.index_cap) return fail(ctx, B200VIS_ERR_CAPACITY, "cluster index list overflow: %u > max_cluster_indices %u", *total, ctx->cl.index_cap);
    if (indices) {
        if (*total > indices_capacity) return fail(ctx, B200VIS_ERR_CAPACITY, "download_clusters: %u indices > capacity %u", *total, indices_capacity);
        CU(cudaMemcpyAsync(indices, ctx->cl.indices + (size_t)view * ctx->cl.index_cap, (size_t)*total * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    return B200VIS_OK;
}

// ---- SURVEY 8(f) N3: check_point_light_mesh_visibility (point lights) ------------------------------------------------
extern "C" int32_t b200vis_enable_visible_diff(b200vis_ctx *ctx, int32_t enabled);
extern "C" int32_t b200vis_upload_shadow_casters(b200vis_ctx *ctx, uint32_t first, uint32_t count, const uint8_t *caster) {
    CHECK_CTX();
    if (count && !caster) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_shadow_casters: null");
    int32_t rc = check_range(ctx, first, count, "upload_shadow_casters"); if (rc) return rc;
    if (!ctx->d_caster) CU(dalloc(&ctx->d_caster, ctx->cfg.max_entities));
    // the stage reads each view's VisibleEntities as a bit set: the sets the visible-diff bookkeeping keeps.  Switched on
    // here, with the first column upload, so that the CULL stage of the coming frame already records them.
    if (!ctx->diff_on) { const int32_t rc2 = b200vis_enable_visible_diff(ctx, 1); if (rc2) return rc2; }
    CU(cudaMemcpyAsync(ctx->d_caster + first, caster, count, cudaMemcpyHostToDevice, ctx->stream));
    return B200VIS_OK;
}
// diff_slots: the items' diff slots (validated), nullptr = none
static int32_t install_shadow_items(b200vis_ctx *ctx, uint32_t n_items, uint32_t list_capacity, const uint32_t *diff_slots) {
    if (!list_capacity) list_capacity = std::max<uint32_t>(ctx->cfg.max_entities, 1);
    if (!ctx->diff_on) return fail(ctx, B200VIS_ERR_NOT_READY, "set_shadow_items: the visible-set bookkeeping was switched off after upload_shadow_casters");
    CU(cudaStreamSynchronize(ctx->stream));
    if (n_items > ctx->shadow_cap_lights || list_capacity > ctx->shadow_cap_list) {
        void *old[] = {ctx->d_shadow_lights, ctx->shadow.mask, ctx->shadow.chunk_count, ctx->shadow.lists, ctx->shadow.count, ctx->shadow.active};
        for (void *p : old) if (p) cudaFree(p);
        ctx->d_shadow_lights = nullptr; ctx->shadow = ShadowBufs{};
        const size_t nl = std::max<uint32_t>(n_items, ctx->shadow_cap_lights), lc = std::max<uint32_t>(list_capacity, ctx->shadow_cap_list);
        CU(dalloc(&ctx->d_shadow_lights, nl));
        CU(dalloc(&ctx->shadow.mask, nl * 6 * ctx->vis.words_stride));
        CU(dalloc(&ctx->shadow.chunk_count, nl * 6 * ctx->vis.chunks_stride));
        CU(dalloc(&ctx->shadow.lists, nl * 6 * lc));
        CU(dalloc(&ctx->shadow.count, nl * 6));
        CU(dalloc(&ctx->shadow.active, nl));
        ctx->shadow_cap_lights = (uint32_t)nl; ctx->shadow_cap_list = (uint32_t)lc;
    }
    if (n_items) CU(cudaMemcpy(ctx->d_shadow_lights, ctx->h_shadow.data(), n_items * sizeof(ShadowLight), cudaMemcpyHostToDevice));
    ctx->shadow_emit_ready = false;             // the lists of the last run belong to other items
    ctx->shadow_ext_on = false;                 // every item's RenderLayers blocks 1..3 are empty again
    ctx->shadow.n_lights = n_items; ctx->shadow.lights = ctx->d_shadow_lights; ctx->shadow.caster = ctx->d_caster;
    ctx->shadow.list_cap = ctx->shadow_cap_list;
    if (ctx->sdiff.added) {
        ctx->h_sdiff_slot.assign(n_items, kNoDiffSlot);
        if (diff_slots) std::copy(diff_slots, diff_slots + n_items, ctx->h_sdiff_slot.begin());
        if (n_items) CU(cudaMemcpy(const_cast<uint32_t *>(ctx->sdiff.slot), ctx->h_sdiff_slot.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice));
    }
    return B200VIS_OK;
}
// the item counts a registered sink bounds (nothing is changed when one is exceeded)
static int32_t check_shadow_sink_items(b200vis_ctx *ctx, uint32_t n_items, const char *who) {
    if (ctx->shsink.entities && n_items > ctx->shsink_max_items)
        return fail(ctx, B200VIS_ERR_CAPACITY, "%s: %u items > the shadow entity sink's max_items %u", who, n_items, ctx->shsink_max_items);
    if (ctx->sdiff.added && n_items > ctx->sdiff_max_items)
        return fail(ctx, B200VIS_ERR_CAPACITY, "%s: %u items > the shadow diff sink's max_items %u", who, n_items, ctx->sdiff_max_items);
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_shadow_lights(b200vis_ctx *ctx, uint32_t n_lights, const uint32_t *light_ordinals, const float *frusta,
                                             const uint64_t *layer_mask, int32_t lod_origin_range_index, uint32_t list_capacity) {
    CHECK_CTX_JOIN();
    if (n_lights && (!light_ordinals || !frusta)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_lights: null");
    if (!ctx->d_caster) return fail(ctx, B200VIS_ERR_NOT_READY, "set_shadow_lights: upload the shadow-caster column first");
    { const int32_t rc = check_shadow_sink_items(ctx, n_lights, "set_shadow_lights"); if (rc) return rc; }
    for (uint32_t i = 0; i < n_lights; ++i)
        if (light_ordinals[i] >= ctx->lights.n) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_lights: light ordinal %u >= %u lights", light_ordinals[i], ctx->lights.n);
    ctx->h_shadow.resize(n_lights);
    for (uint32_t i = 0; i < n_lights; ++i) {
        ShadowLight &s = ctx->h_shadow[i];
        memset(&s, 0, sizeof s);
        memcpy(s.planes, frusta + (size_t)i * 144, sizeof s.planes);
        s.layers = layer_mask ? layer_mask[i] : 1ull;
        s.row = ctx->h_light_row[light_ordinals[i]]; s.range = ctx->h_light_range[light_ordinals[i]]; s.kind = 0;
        s.range_index = (lod_origin_range_index >= 0 && lod_origin_range_index < 32) ? lod_origin_range_index : -1;
    }
    return install_shadow_items(ctx, n_lights, list_capacity, nullptr);
}
static int32_t set_shadow_items(b200vis_ctx *ctx, uint32_t n_items, const b200vis_shadow_item *items, uint32_t list_capacity,
                                const uint32_t *diff_slots) {
    if (n_items && !items) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_items: null");
    if (!ctx->d_caster) return fail(ctx, B200VIS_ERR_NOT_READY, "set_shadow_items: upload the shadow-caster column first");
    { const int32_t rc = check_shadow_sink_items(ctx, n_items, "set_shadow_items"); if (rc) return rc; }
    ctx->h_shadow.resize(n_items);
    for (uint32_t i = 0; i < n_items; ++i) {
        const b200vis_shadow_item &it = items[i];
        if (it.kind > B200VIS_SHADOW_DIRECTIONAL_CASCADE) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_items: item %u has kind %u", i, it.kind);
        if (it.kind != B200VIS_SHADOW_DIRECTIONAL_CASCADE && (it.light_row >= ctx->n || row_is_dead(ctx, it.light_row)))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_items: item %u: light row %u out of range or despawned", i, it.light_row);
        ShadowLight &s = ctx->h_shadow[i];
        memset(&s, 0, sizeof s);
        memcpy(s.planes, it.frusta, sizeof s.planes);
        s.layers = it.layer_mask; s.row = it.kind == B200VIS_SHADOW_DIRECTIONAL_CASCADE ? 0u : it.light_row; s.range = it.range;
        s.kind = it.kind; s.range_index = (it.range_view_index >= 0 && it.range_view_index < 32) ? it.range_view_index : -1;
    }
    return install_shadow_items(ctx, n_items, list_capacity, diff_slots);
}
extern "C" int32_t b200vis_set_shadow_items(b200vis_ctx *ctx, uint32_t n_items, const b200vis_shadow_item *items, uint32_t list_capacity) {
    CHECK_CTX_JOIN();
    return set_shadow_items(ctx, n_items, items, list_capacity, nullptr);
}
extern "C" int32_t b200vis_set_shadow_items_ex(b200vis_ctx *ctx, uint32_t n_items, const b200vis_shadow_item *items, uint32_t list_capacity,
                                               const uint32_t *diff_slots) {
    CHECK_CTX_JOIN();
    if (diff_slots) {
        if (!ctx->sdiff.added) return fail(ctx, B200VIS_ERR_NOT_READY, "set_shadow_items_ex: diff slots without a shadow diff sink");
        std::vector<uint8_t> seen(ctx->sdiff_max_slots, 0);
        for (uint32_t i = 0; i < n_items; ++i) {
            const uint32_t s = diff_slots[i];
            if (s == B200VIS_SHADOW_NO_SLOT) continue;
            if (s >= ctx->sdiff_max_slots)
                return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_items_ex: item %u: slot %u >= max_slots %u", i, s, ctx->sdiff_max_slots);
            if (seen[s]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_items_ex: slot %u named twice", s);
            seen[s] = 1;
        }
    }
    return set_shadow_items(ctx, n_items, items, list_capacity, diff_slots);
}
extern "C" int32_t b200vis_run_shadow_culling(b200vis_ctx *ctx) {
    CHECK_CTX_JOIN();   // reads what the frame's CULL stage (incl. its tail on the side stream) left behind
    if (!ctx->d_caster || !ctx->diff.prev) return fail(ctx, B200VIS_ERR_NOT_READY, "run_shadow_culling: call b200vis_set_shadow_lights first");
    if (ctx->frame == 0) return fail(ctx, B200VIS_ERR_NOT_READY, "run_shadow_culling: run the CULL stage first");
    cudaStream_t st = ctx->stream;
    if (ctx->sdiff.added) {
        // a slot no item of this run names is emptied (the render world drops an unextracted light's lists): only the ones
        // that may hold entries, so a steady frame clears nothing.  An inactive item's slot is emptied by the expansion.
        std::vector<uint8_t> named(ctx->sdiff_max_slots, 0);
        for (uint32_t i = 0; i < ctx->shadow.n_lights; ++i)
            if (ctx->h_sdiff_slot[i] != kNoDiffSlot) named[ctx->h_sdiff_slot[i]] = 1;
        const size_t ws = ctx->vis.words_stride, cs = ctx->vis.chunks_stride;
        for (uint32_t s = 0; s < ctx->sdiff_max_slots; ++s) {
            if (ctx->sdiff_held[s] && !named[s]) {
                CU(cudaMemsetAsync(ctx->sdiff.prev + (size_t)s * 6 * ws, 0, 6 * ws * 4, st));
                CU(cudaMemsetAsync(ctx->sdiff.prev_count + (size_t)s * 6 * cs, 0, 6 * cs * 4, st));
            }
            ctx->sdiff_held[s] = named[s];
        }
    }
    ctx->shadow_emit_ready = false;
    if (!ctx->shadow.n_lights) {                // the sinks' one offset: a memset, no launch
        ctx->shadow_emit_ready = ctx->shsink.entities != nullptr;
        if (ctx->shsink.entities) CU(cudaMemsetAsync(ctx->shsink.offsets, 0, 4, st));
        if (ctx->sdiff.added) {
            CU(cudaMemsetAsync(ctx->sdiff.added_offsets, 0, 4, st));
            CU(cudaMemsetAsync(ctx->sdiff.removed_offsets, 0, 4, st));
        }
        return B200VIS_OK;
    }
    Rows R = ctx->rows;
    R.layers = ctx->have_layers ? ctx->d_layers : nullptr;
    R.range = ctx->have_range ? ctx->d_range : nullptr;
    R.rank = ctx->rank_identity ? nullptr : ctx->d_rank;
    R.row_of_rank = ctx->rank_identity ? nullptr : ctx->d_row_of_rank;
    ShadowBufs sb = ctx->shadow;
    sb.has_ranges = ctx->have_range ? 1u : 0u;
    if (ctx->shadow_ext_on && ctx->have_layers_ext) {   // blocks 1..3 on both sides: k_shadow_cull<true>
        sb.layers_ext = ctx->d_shadow_layers_ext;
        R.layers_ext = ctx->d_layers_ext;
    }
    CU(cudaMemsetAsync(sb.chunk_count, 0, (size_t)sb.n_lights * 6 * ctx->vis.chunks_stride * 4, st));
    ShadowSink sink = ctx->shsink;
    sink.keys = ctx->d_keys;                    // a compaction swaps the key buffers
    ShadowDiff sd = ctx->sdiff;
    sd.keys = ctx->d_keys;
    // with an entity sink, keep the masks for b200vis_emit_shadow_entities (a sink too small for this run is grown and
    // filled from them)
    const size_t kept = ctx->shsink.entities ? (size_t)sb.n_lights * 6 * ctx->vis.words_stride : 0;
    if (kept > ctx->shadow_kept_cap) {
        if (ctx->d_shadow_kept) cudaFree(ctx->d_shadow_kept);
        ctx->d_shadow_kept = nullptr; ctx->shadow_kept_cap = 0;
        CU(dalloc(&ctx->d_shadow_kept, (size_t)ctx->shadow_cap_lights * 6 * ctx->vis.words_stride));
        ctx->shadow_kept_cap = (size_t)ctx->shadow_cap_lights * 6 * ctx->vis.words_stride;
    }
    CU(launch_shadow_cull(st, R, sb, ctx->diff.prev, active_consts(ctx).n_views, ctx->vis.n_words, ctx->vis.n_chunks,
                          ctx->vis.words_stride, ctx->vis.chunks_stride, ctx->d_stats, (ctx->frame + 2u) % 3u, sink, sd,
                          kept ? ctx->d_shadow_kept : nullptr));
    CU(cudaGetLastError());
    ctx->shadow_emit_ready = kept != 0;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_emit_shadow_entities(b200vis_ctx *ctx) {
    CHECK_CTX_JOIN();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "emit_shadow_entities: world_size > 1");
    if (!ctx->shsink.entities) return fail(ctx, B200VIS_ERR_NOT_READY, "emit_shadow_entities: no shadow entity sink registered");
    if (!ctx->shadow_emit_ready)
        return fail(ctx, B200VIS_ERR_NOT_READY, "emit_shadow_entities: no b200vis_run_shadow_culling with an entity sink since the items "
                    "or the topology were last set");
    // registering a sink and installing items both refuse this combination already; checked again because the expansion
    // would write past the sink's offsets otherwise
    if (ctx->shsink_max_items < ctx->shadow.n_lights)
        return fail(ctx, B200VIS_ERR_CAPACITY, "emit_shadow_entities: max_items %u < %u installed shadow items", ctx->shsink_max_items,
                    ctx->shadow.n_lights);
    cudaStream_t st = ctx->stream;
    if (!ctx->shadow.n_lights) { CU(cudaMemsetAsync(ctx->shsink.offsets, 0, 4, st)); return B200VIS_OK; }
    ShadowSink sink = ctx->shsink;
    sink.keys = ctx->d_keys;
    CU(launch_emit_shadow_entities(st, ctx->shadow, ctx->d_shadow_kept, ctx->rows.n, ctx->vis.n_words, ctx->vis.n_chunks,
                                   ctx->vis.words_stride, ctx->vis.chunks_stride, ctx->rank_identity ? nullptr : ctx->d_row_of_rank, sink));
    CU(cudaGetLastError());
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_shadow_visible(b200vis_ctx *ctx, uint32_t shadow_light, uint32_t face, uint32_t *rows, uint32_t capacity,
                                                   uint32_t *count) {
    CHECK_CTX_JOIN();
    if (shadow_light >= ctx->shadow.n_lights || face >= 6 || !count) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_shadow_visible: bad argument");
    cudaStream_t st = ctx->stream;
    const uint32_t list = shadow_light * 6 + face;
    uint32_t c = 0;
    CU(cudaMemcpyAsync(&c, ctx->shadow.count + list, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    *count = c;
    if (rows) {
        if (c > capacity || c > ctx->shadow.list_cap)
            return fail(ctx, B200VIS_ERR_CAPACITY, "download_shadow_visible: %u rows > capacity %u (list capacity %u)", c, capacity, ctx->shadow.list_cap);
        if (c) CU(cudaMemcpyAsync(rows, ctx->shadow.lists + (size_t)list * ctx->shadow.list_cap, (size_t)c * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    return B200VIS_OK;
}

static int32_t map_host(b200vis_ctx *ctx, void *p, size_t bytes, uint32_t **dev);
extern "C" int32_t b200vis_set_shadow_entities_sink(b200vis_ctx *ctx, const b200vis_shadow_entities_sink *sink) {
    CHECK_CTX_JOIN();
    if (sink) {
        if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_shadow_entities_sink: world_size > 1");
        if (!sink->entities || !sink->offsets || !sink->active || !sink->capacity)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_entities_sink: entities, offsets, active and a capacity go together");
        if (reinterpret_cast<uintptr_t>(sink->entities) & 7u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_entities_sink: entities is not 8-byte aligned");
        if (sink->max_items < ctx->shadow.n_lights)
            return fail(ctx, B200VIS_ERR_CAPACITY, "set_shadow_entities_sink: max_items %u < %u installed shadow items", sink->max_items,
                        ctx->shadow.n_lights);
    }
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->shsink = ShadowSink{}; ctx->shsink_max_items = 0;
    if (!sink) return B200VIS_OK;
    const size_t n_off = (size_t)sink->max_items * 6 + 1;
    int32_t rc;
    uint32_t *de = nullptr, *doff = nullptr, *dact = nullptr;
    if ((rc = map_host(ctx, sink->entities, (size_t)sink->capacity * 8, &de))) return rc;
    if ((rc = map_host(ctx, sink->offsets, n_off * 4, &doff))) return rc;
    if ((rc = map_host(ctx, sink->active, std::max<size_t>(sink->max_items, 1), &dact))) return rc;
    if (n_off > ctx->shadow_off_cap) {
        if (ctx->d_shadow_off) cudaFree(ctx->d_shadow_off);
        ctx->d_shadow_off = nullptr; ctx->shadow_off_cap = 0;
        CU(dalloc(&ctx->d_shadow_off, n_off));
        ctx->shadow_off_cap = n_off;
    }
    if ((rc = make_keys_resident(ctx))) return rc;
    ShadowSink &s = ctx->shsink;
    s.entities = reinterpret_cast<uint64_t *>(de); s.capacity = sink->capacity; s.offsets = doff;
    s.active = reinterpret_cast<uint8_t *>(dact); s.dev_offsets = ctx->d_shadow_off;
    ctx->shsink_max_items = sink->max_items;
    return B200VIS_OK;
}

static void free_shadow_diff(b200vis_ctx *ctx) {
    ShadowDiff &d = ctx->sdiff;
    for (void *p : {(void *)d.slot, (void *)d.prev, (void *)d.prev_count, (void *)d.words, (void *)d.chunk, (void *)d.dev_offsets})
        if (p) cudaFree(p);
    d = ShadowDiff{}; ctx->sdiff_max_items = ctx->sdiff_max_slots = 0;
    ctx->h_sdiff_slot.clear(); ctx->sdiff_held.clear();
}
extern "C" int32_t b200vis_set_shadow_diff_sink(b200vis_ctx *ctx, const b200vis_shadow_diff_sink *sink) {
    CHECK_CTX_JOIN();
    if (sink) {
        if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_shadow_diff_sink: world_size > 1");
        if (!sink->added || !sink->removed || !sink->added_offsets || !sink->removed_offsets || !sink->added_capacity || !sink->removed_capacity)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_diff_sink: added, removed, both offsets and both capacities go together");
        if ((reinterpret_cast<uintptr_t>(sink->added) | reinterpret_cast<uintptr_t>(sink->removed)) & 7u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_shadow_diff_sink: added / removed is not 8-byte aligned");
        if (sink->max_items < ctx->shadow.n_lights)
            return fail(ctx, B200VIS_ERR_CAPACITY, "set_shadow_diff_sink: max_items %u < %u installed shadow items", sink->max_items,
                        ctx->shadow.n_lights);
    }
    CU(cudaStreamSynchronize(ctx->stream));
    free_shadow_diff(ctx);
    if (!sink) return B200VIS_OK;
    const size_t n_off = (size_t)sink->max_items * 6 + 1, ws = ctx->vis.words_stride, cs = ctx->vis.chunks_stride;
    const size_t lists = std::max<size_t>(sink->max_items, 1) * 6;
    int32_t rc;
    uint32_t *da = nullptr, *dr = nullptr, *dao = nullptr, *dro = nullptr;
    if ((rc = map_host(ctx, sink->added, (size_t)sink->added_capacity * 8, &da))) return rc;
    if ((rc = map_host(ctx, sink->removed, (size_t)sink->removed_capacity * 8, &dr))) return rc;
    if ((rc = map_host(ctx, sink->added_offsets, n_off * 4, &dao))) return rc;
    if ((rc = map_host(ctx, sink->removed_offsets, n_off * 4, &dro))) return rc;
    if ((rc = make_keys_resident(ctx))) return rc;
    ShadowDiff &d = ctx->sdiff;
    uint32_t *slot = nullptr;
    const cudaError_t e = [&]() {
        cudaError_t x;
        if ((x = dalloc(&slot, sink->max_items)) != cudaSuccess) return x;
        d.slot = slot;
        if ((x = dalloc(&d.prev, (size_t)sink->max_slots * 6 * ws)) != cudaSuccess) return x;          // every slot empty
        if ((x = dalloc(&d.prev_count, (size_t)sink->max_slots * 6 * cs)) != cudaSuccess) return x;
        if ((x = dalloc(&d.words, 2 * lists * ws)) != cudaSuccess) return x;
        if ((x = dalloc(&d.chunk, lists * cs)) != cudaSuccess) return x;
        return dalloc(&d.dev_offsets, 2 * (lists + 1));
    }();
    if (e != cudaSuccess) {
        cudaGetLastError();
        free_shadow_diff(ctx);
        return fail(ctx, e == cudaErrorMemoryAllocation ? B200VIS_ERR_OUT_OF_MEMORY : B200VIS_ERR_CUDA, "set_shadow_diff_sink: %zu slot sets: %s",
                    (size_t)sink->max_slots * 6, cudaGetErrorString(e));
    }
    d.lists = (uint32_t)lists;
    d.added = reinterpret_cast<uint64_t *>(da); d.removed = reinterpret_cast<uint64_t *>(dr);
    d.added_capacity = sink->added_capacity; d.removed_capacity = sink->removed_capacity;
    d.added_offsets = dao; d.removed_offsets = dro;
    ctx->sdiff_max_items = sink->max_items; ctx->sdiff_max_slots = sink->max_slots;
    ctx->sdiff_held.assign(sink->max_slots, 0);
    ctx->h_sdiff_slot.assign(ctx->shadow.n_lights, kNoDiffSlot);   // the installed items have no slot until they are set again
    if (ctx->shadow.n_lights) CU(cudaMemset(slot, 0xFF, (size_t)ctx->shadow.n_lights * 4));
    return B200VIS_OK;
}

static void free_view_diff(ViewDiff &d) {
    for (void *p : {(void *)d.prev, (void *)d.prev_count, (void *)d.words, (void *)d.chunk, (void *)d.dev_offsets})
        if (p) cudaFree(p);
    d = ViewDiff{};
}
extern "C" int32_t b200vis_set_view_diff_sink(b200vis_ctx *ctx, const b200vis_view_diff_sink *sink) {
    CHECK_CTX_JOIN();
    if (sink) {
        if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_view_diff_sink: world_size > 1");
        if (!sink->added || !sink->removed || !sink->added_offsets || !sink->removed_offsets || !sink->added_capacity || !sink->removed_capacity)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_view_diff_sink: added, removed, both offsets and both capacities go together");
        if ((reinterpret_cast<uintptr_t>(sink->added) | reinterpret_cast<uintptr_t>(sink->removed)) & 7u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_view_diff_sink: added / removed is not 8-byte aligned");
    }
    CU(cudaStreamSynchronize(ctx->stream));
    if (!sink) {
        free_view_diff(ctx->vdiff); ctx->vdiff_max_slots = 0;
        ctx->h_vdiff_slot.clear(); ctx->vdiff_held.clear();
        return B200VIS_OK;
    }
    const size_t lists = (size_t)ctx->cfg.max_views * 8, ws = ctx->vis.words_stride, cs = ctx->vis.chunks_stride;
    const size_t sets = (size_t)std::max<uint32_t>(sink->max_slots, 1) * 8;
    int32_t rc;
    uint32_t *da = nullptr, *dr = nullptr, *dao = nullptr, *dro = nullptr;
    if ((rc = map_host(ctx, sink->added, (size_t)sink->added_capacity * 8, &da))) return rc;
    if ((rc = map_host(ctx, sink->removed, (size_t)sink->removed_capacity * 8, &dr))) return rc;
    if ((rc = map_host(ctx, sink->added_offsets, (lists + 1) * 4, &dao))) return rc;
    if ((rc = map_host(ctx, sink->removed_offsets, (lists + 1) * 4, &dro))) return rc;
    ViewDiff d{};
    const cudaError_t e = [&]() {
        cudaError_t x;
        if ((x = dalloc(&d.prev, sets * ws)) != cudaSuccess) return x;              // every slot empty
        if ((x = dalloc(&d.prev_count, sets / 8 * cs)) != cudaSuccess) return x;
        if ((x = dalloc(&d.words, 2 * sets * ws)) != cudaSuccess) return x;
        if ((x = dalloc(&d.chunk, sets * cs)) != cudaSuccess) return x;
        return dalloc(&d.dev_offsets, 2 * (lists + 1));
    }();
    if (e != cudaSuccess) {
        cudaGetLastError();
        free_view_diff(d);
        return fail(ctx, e == cudaErrorMemoryAllocation ? B200VIS_ERR_OUT_OF_MEMORY : B200VIS_ERR_CUDA, "set_view_diff_sink: %zu slot sets: %s",
                    sets, cudaGetErrorString(e));
    }
    if ((rc = make_keys_resident(ctx))) { free_view_diff(d); return rc; }
    d.sets = (uint32_t)sets; d.lists = (uint32_t)lists;
    d.added = reinterpret_cast<uint64_t *>(da); d.removed = reinterpret_cast<uint64_t *>(dr);
    d.added_capacity = sink->added_capacity; d.removed_capacity = sink->removed_capacity;
    d.added_offsets = dao; d.removed_offsets = dro;
    free_view_diff(ctx->vdiff);
    ctx->vdiff = d; ctx->vdiff_max_slots = sink->max_slots;
    ctx->vdiff_held.assign(sink->max_slots, 0);
    ctx->h_vdiff_slot.assign(ctx->cfg.max_views, kNoDiffSlot);   // no view has a slot until the slots are set
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_view_diff_slots(b200vis_ctx *ctx, uint32_t n_views, const uint32_t *slots) {
    CHECK_CTX();
    if (n_views > ctx->cfg.max_views) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_view_diff_slots: %u views > max_views %u", n_views, ctx->cfg.max_views);
    if (n_views && !slots) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_view_diff_slots: null");
    if (!ctx->vdiff.added) return fail(ctx, B200VIS_ERR_NOT_READY, "set_view_diff_slots: no view diff sink is registered");
    std::vector<uint8_t> seen(ctx->vdiff_max_slots, 0);
    for (uint32_t v = 0; v < n_views; ++v) {
        const uint32_t s = slots[v];
        if (s == B200VIS_VIEW_NO_SLOT) continue;
        if (s >= ctx->vdiff_max_slots)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_view_diff_slots: view %u: slot %u >= max_slots %u", v, s, ctx->vdiff_max_slots);
        if (seen[s]) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_view_diff_slots: slot %u named twice", s);
        seen[s] = 1;
    }
    std::fill(ctx->h_vdiff_slot.begin(), ctx->h_vdiff_slot.end(), kNoDiffSlot);
    std::copy(slots, slots + n_views, ctx->h_vdiff_slot.begin());
    return B200VIS_OK;
}

// ---- SURVEY 8(f) N4: check_visibility_ranges and visibility_propagate_system --------------------------------------
extern "C" int32_t b200vis_upload_visibility_ranges(b200vis_ctx *ctx, uint32_t first, uint32_t count, const float *start_end,
                                                    const uint8_t *use_aabb) {
    CHECK_CTX();
    if (count && (!start_end || !use_aabb)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_visibility_ranges: null");
    int32_t rc = check_range(ctx, first, count, "upload_visibility_ranges"); if (rc) return rc;
    if (!ctx->d_range_se) {
        CU(dalloc(&ctx->d_range_se, ctx->cfg.max_entities));
        CU(dalloc(&ctx->d_range_ua, ctx->cfg.max_entities));
        CU(dalloc(&ctx->d_range_views, 32));
    }
    const size_t ou = (size_t)count * 8;
    rc = stage_in(ctx, start_end, (size_t)count * 8, 0); if (rc) return rc;
    rc = stage_in(ctx, use_aabb, count, ou); if (rc) return rc;
    launch_unpack_range_params(ctx->stream, ctx->d_range_se, ctx->d_range_ua, first, count,
                               reinterpret_cast<const float *>(ctx->d_stage), ctx->d_stage + ou);
    CU(cudaGetLastError());
    ctx->have_range = true;   // the cull kernels now take the non-SIMPLE path and fill d_range themselves
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_visibility_range_views(b200vis_ctx *ctx, uint32_t n_views, const float *positions) {
    CHECK_CTX();
    if (n_views && !positions) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_visibility_range_views: null");
    if (!ctx->d_range_views) return fail(ctx, B200VIS_ERR_NOT_READY, "set_visibility_range_views: upload the VisibilityRange columns first");
    if (n_views > 32) n_views = 32;   // view_query.iter().take(32) (range.rs:247)
    float4 h[32];
    for (uint32_t v = 0; v < n_views; ++v) h[v] = make_float4(positions[v * 3], positions[v * 3 + 1], positions[v * 3 + 2], 0.0f);
    // pageable source: the copy is staged before the call returns, and is ordered before the next frame on the stream
    if (n_views) CU(cudaMemcpyAsync(ctx->d_range_views, h, n_views * sizeof(float4), cudaMemcpyHostToDevice, ctx->stream));
    ctx->n_range_views = n_views;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_visibility_ranges(b200vis_ctx *ctx, uint32_t first, uint32_t count, uint32_t *mask) {
    CHECK_CTX_JOIN();
    if (count && !mask) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_visibility_ranges: null");
    int32_t rc = check_range(ctx, first, count, "download_visibility_ranges"); if (rc) return rc;
    if (!ctx->have_range) return fail(ctx, B200VIS_ERR_NOT_READY, "download_visibility_ranges: no VisibilityRange data was uploaded");
    Rows R = ctx->rows; R.range = ctx->d_range;
    launch_pack_ranges(ctx->stream, R, first, count, reinterpret_cast<uint32_t *>(ctx->d_stage));
    CU(cudaMemcpyAsync(mask, ctx->d_stage, (size_t)count * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_upload_visibility(b200vis_ctx *ctx, uint32_t first, uint32_t count, const uint8_t *visibility) {
    CHECK_CTX();
    if (count && !visibility) return fail(ctx, B200VIS_ERR_INVALID_ARG, "upload_visibility: null");
    int32_t rc = check_range(ctx, first, count, "upload_visibility"); if (rc) return rc;
    if (!ctx->d_visibility) {   // rows never uploaded: Visibility::Inherited (the component default)
        CU(dalloc(&ctx->d_visibility, ctx->cfg.max_entities));
        CU(dalloc(&ctx->d_iv_changed, ctx->cfg.max_entities));
    }
    CU(cudaMemcpyAsync(ctx->d_visibility + first, visibility, count, cudaMemcpyHostToDevice, ctx->stream));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_propagate_visibility(b200vis_ctx *ctx) {
    CHECK_CTX_JOIN();   // the tail of an earlier frame may still read the flags column
    if (!ctx->topology_set) return fail(ctx, B200VIS_ERR_NOT_READY, "propagate_visibility: set_topology first");
    if (!ctx->d_visibility) return fail(ctx, B200VIS_ERR_NOT_READY, "propagate_visibility: upload the Visibility column first");
    const uint32_t n_pass = ctx->pass_begin.empty() ? 0 : (uint32_t)ctx->pass_begin.size() - 1;
    for (uint32_t p = 0; p < n_pass; ++p)
        launch_visibility_propagate(ctx->stream, ctx->rows, ctx->d_tiles + ctx->pass_begin[p], ctx->pass_begin[p + 1] - ctx->pass_begin[p],
                                    ctx->d_visibility, ctx->d_iv_changed);
    CU(cudaGetLastError());
    ctx->iv_ran = true;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_inherited_visibility(b200vis_ctx *ctx, uint32_t first, uint32_t count, uint8_t *inherited, uint8_t *changed) {
    CHECK_CTX_JOIN();
    int32_t rc = check_range(ctx, first, count, "download_inherited_visibility"); if (rc) return rc;
    cudaStream_t st = ctx->stream;
    launch_pack_inherited(st, ctx->rows, first, count, ctx->iv_ran ? ctx->d_iv_changed : nullptr, ctx->d_stage);
    if (inherited) CU(cudaMemcpyAsync(inherited, ctx->d_stage, count, cudaMemcpyDeviceToHost, st));
    if (changed) CU(cudaMemcpyAsync(changed, ctx->d_stage + count, count, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return B200VIS_OK;
}

// ---- SURVEY 8(f) N2: Clusters -> ViewClusterBindings buffers ---------------------------------------------------
extern "C" int32_t b200vis_set_cluster_bindings(b200vis_ctx *ctx, uint32_t mode, const uint32_t *gpu_index_of_light, uint32_t n_map) {
    CHECK_CTX_JOIN();
    if (mode > B200VIS_BINDINGS_UNIFORM) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_cluster_bindings: mode %u", mode);
    if (gpu_index_of_light && !n_map) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_cluster_bindings: empty index map");
    const size_t V = ctx->cfg.max_views;
    if (mode && !ctx->bind.oc) {
        ctx->bind.il_stride = std::max<uint32_t>(ctx->cl.index_cap, 4096u);
        CU(dalloc(&ctx->bind.oc, V * kMaxClusters * 8));
        CU(dalloc(&ctx->bind.il, V * (size_t)ctx->bind.il_stride));
        CU(dalloc(&ctx->bind.count, V * 2));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    if (gpu_index_of_light) {
        if (n_map > ctx->bind_map_cap) {
            if (ctx->d_bind_map) cudaFree(ctx->d_bind_map);
            ctx->d_bind_map = nullptr; ctx->bind_map_cap = n_map;
            CU(dalloc(&ctx->d_bind_map, n_map));
        }
        CU(cudaMemcpy(ctx->d_bind_map, gpu_index_of_light, (size_t)n_map * 4, cudaMemcpyHostToDevice));
        ctx->bind.map = ctx->d_bind_map; ctx->bind.n_map = n_map;
    } else { ctx->bind.map = nullptr; ctx->bind.n_map = 0; }
    ctx->bind.mode = mode;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_cluster_bindings(b200vis_ctx *ctx, uint32_t view, uint32_t *offsets_and_counts, uint32_t oc_capacity,
                                                     uint32_t *index_lists, uint32_t il_capacity, uint32_t *n_offsets, uint32_t *n_indices) {
    CHECK_CTX_JOIN();
    if (view >= ctx->cfg.max_views || !n_offsets || !n_indices) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_cluster_bindings: bad argument");
    if (!ctx->bind.mode) return fail(ctx, B200VIS_ERR_NOT_READY, "download_cluster_bindings: call b200vis_set_cluster_bindings first");
    cudaStream_t st = ctx->stream;
    uint32_t cnt[2] = {0, 0};
    CU(cudaMemcpyAsync(cnt, ctx->bind.count + view * 2, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    *n_offsets = cnt[0]; *n_indices = cnt[1];
    const bool storage = ctx->bind.mode == B200VIS_BINDINGS_STORAGE;
    const uint32_t oc_words = storage ? cnt[0] * 8u : 4096u, il_words = storage ? cnt[1] : 4096u;
    if ((offsets_and_counts && oc_words > oc_capacity) || (index_lists && il_words > il_capacity))
        return fail(ctx, B200VIS_ERR_CAPACITY, "download_cluster_bindings: needs %u + %u words, capacities %u + %u", oc_words, il_words, oc_capacity, il_capacity);
    if (offsets_and_counts && oc_words)
        CU(cudaMemcpyAsync(offsets_and_counts, ctx->bind.oc + (size_t)view * kMaxClusters * 8, (size_t)oc_words * 4, cudaMemcpyDeviceToHost, st));
    if (index_lists && il_words)
        CU(cudaMemcpyAsync(index_lists, ctx->bind.il + (size_t)view * ctx->bind.il_stride, (size_t)il_words * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return B200VIS_OK;
}

// ---- SURVEY 8(f) N1: added / removed rows of each view's VisibleEntities against last frame -----------------
static int32_t reset_visible_diff(b200vis_ctx *ctx) {
    if (ctx->diff.prev)
        CU(cudaMemsetAsync(ctx->diff.prev, 0, (size_t)ctx->vis.words_stride * ctx->cfg.max_views * 4, ctx->stream));
    return B200VIS_OK;
}
extern "C" int32_t b200vis_enable_visible_diff(b200vis_ctx *ctx, int32_t enabled) {
    CHECK_CTX_JOIN();
    if (enabled && !ctx->diff.prev) {
        const size_t V = ctx->cfg.max_views, W = ctx->vis.words_stride;
        CU(dalloc(&ctx->diff.prev, W * V));
        CU(dalloc(&ctx->diff.words, 2 * W * V));
        CU(dalloc(&ctx->diff.chunk, (size_t)ctx->vis.chunks_stride * V));
        CU(dalloc(&ctx->diff.lists, 2 * (size_t)ctx->vis.list_stride * V));
        CU(dalloc(&ctx->diff.count, 2 * V));
    }
    if (enabled && !ctx->diff_on) { const int32_t rc = reset_visible_diff(ctx); if (rc) return rc; }   // old list = empty
    ctx->diff_on = enabled != 0;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_download_visible_diff(b200vis_ctx *ctx, uint32_t view, uint32_t *added_rows, uint32_t added_capacity,
                                                 uint32_t *n_added, uint32_t *removed_rows, uint32_t removed_capacity,
                                                 uint32_t *n_removed) {
    CHECK_CTX_JOIN();
    if (view >= ctx->cfg.max_views || !n_added || !n_removed) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_visible_diff: bad argument");
    if (!ctx->diff_on) return fail(ctx, B200VIS_ERR_NOT_READY, "download_visible_diff: call b200vis_enable_visible_diff first");
    cudaStream_t st = ctx->stream;
    uint32_t cnt[2] = {0, 0};
    CU(cudaMemcpyAsync(cnt, ctx->diff.count + view * 2, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    *n_added = cnt[0]; *n_removed = cnt[1];
    if ((added_rows && cnt[0] > added_capacity) || (removed_rows && cnt[1] > removed_capacity))
        return fail(ctx, B200VIS_ERR_CAPACITY, "download_visible_diff: %u added / %u removed rows exceed the capacities %u / %u",
                    cnt[0], cnt[1], added_capacity, removed_capacity);
    const size_t V = ctx->cfg.max_views, LS = ctx->vis.list_stride;
    if (added_rows && cnt[0]) CU(cudaMemcpyAsync(added_rows, ctx->diff.lists + (size_t)view * LS, (size_t)cnt[0] * 4, cudaMemcpyDeviceToHost, st));
    if (removed_rows && cnt[1]) CU(cudaMemcpyAsync(removed_rows, ctx->diff.lists + (V + view) * LS, (size_t)cnt[1] * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return B200VIS_OK;
}

static int32_t map_host(b200vis_ctx *ctx, void *p, size_t bytes, uint32_t **dev);
extern "C" int32_t b200vis_set_visible_diff_sink(b200vis_ctx *ctx, uint32_t *rows, uint32_t capacity, uint32_t *counts) {
    CHECK_CTX_JOIN();
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->diff_sink_rows_d = ctx->diff_sink_counts_d = nullptr; ctx->diff_sink_cap = 0;
    if (!rows && !counts) return B200VIS_OK;
    if (!rows || !counts || !capacity) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_visible_diff_sink: rows, counts and a capacity go together");
    const size_t V = ctx->cfg.max_views;
    int32_t rc;
    uint32_t *dr = nullptr, *dc = nullptr;
    if ((rc = map_host(ctx, rows, 2 * V * (size_t)capacity * 4, &dr))) return rc;
    if ((rc = map_host(ctx, counts, 2 * V * 4, &dc))) return rc;
    ctx->diff_sink_rows_d = dr; ctx->diff_sink_counts_d = dc; ctx->diff_sink_cap = capacity;
    return B200VIS_OK;
}

static int32_t map_host(b200vis_ctx *ctx, void *p, size_t bytes, uint32_t **dev) {
    *dev = nullptr;
    if (!p) return B200VIS_OK;
    // already pinned (cudaHostAlloc / a previous cudaHostRegister, e.g. torch pinned tensors): UVA gives the device alias
    void *d = nullptr;
    if (cudaHostGetDevicePointer(&d, p, 0) != cudaSuccess) {
        cudaGetLastError();
        cudaError_t e = cudaHostRegister(p, bytes, cudaHostRegisterMapped | cudaHostRegisterPortable);
        if (e != cudaSuccess && e != cudaErrorHostMemoryAlreadyRegistered)
            return fail(ctx, B200VIS_ERR_CUDA, "set_result_sink: memory is not pinned and cudaHostRegister failed: %s", cudaGetErrorString(e));
        cudaGetLastError();
        CU(cudaHostGetDevicePointer(&d, p, 0));
    }
    *dev = static_cast<uint32_t *>(d);
    return B200VIS_OK;
}
extern "C" int32_t b200vis_set_result_sink(b200vis_ctx *ctx, const b200vis_result_sink *sink) {
    CHECK_CTX_JOIN();
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->have_sink = false;
    if (!sink) return B200VIS_OK;
    if (!sink->stats) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_result_sink: stats is required");
    const size_t V = ctx->cfg.max_views;
    int32_t rc;
    if ((rc = map_host(ctx, sink->stats, sizeof(b200vis_frame_stats), &ctx->sink_stats_d))) return rc;
    if ((rc = map_host(ctx, sink->visible_rows, V * sink->visible_capacity * 4, &ctx->sink_rows_d))) return rc;
    { uint32_t *d = nullptr; if ((rc = map_host(ctx, sink->visible_classes, V * (size_t)sink->visible_capacity, &d))) return rc; ctx->sink_cls_d = reinterpret_cast<uint8_t *>(d); }
    if ((rc = map_host(ctx, sink->cluster_offsets, V * (kMaxClusters + 1) * 4, &ctx->sink_off_d))) return rc;
    if ((rc = map_host(ctx, sink->cluster_indices, V * (size_t)sink->cluster_capacity * 4, &ctx->sink_idx_d))) return rc;
    if ((sink->cluster_offsets == nullptr) != (sink->cluster_indices == nullptr))
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_result_sink: cluster_offsets and cluster_indices go together");
    ctx->sink = *sink;
    ctx->have_sink = true;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_view_stats_sink(b200vis_ctx *ctx, uint32_t *per_view) {
    CHECK_CTX_JOIN();
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->view_stats_sink = ctx->view_stats_d = nullptr;
    if (!per_view) return B200VIS_OK;
    const int32_t rc = map_host(ctx, per_view, (size_t)ctx->cfg.max_views * 16, &ctx->view_stats_d); if (rc) return rc;
    ctx->view_stats_sink = per_view;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_visible_entities_sink(b200vis_ctx *ctx, const b200vis_visible_entities_sink *sink) {
    CHECK_CTX_JOIN();
    if (sink) {
        if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_visible_entities_sink: world_size > 1");
        if (!sink->entities || !sink->offsets || !sink->capacity)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_visible_entities_sink: entities, offsets and a capacity go together");
        if (reinterpret_cast<uintptr_t>(sink->entities) & 7u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_visible_entities_sink: entities is not 8-byte aligned");
    }
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->ent_sink_d = nullptr; ctx->ent_off_d = nullptr; ctx->ent_cap = 0;
    if (!sink) return B200VIS_OK;
    const size_t V = ctx->cfg.max_views;
    int32_t rc;
    uint32_t *de = nullptr, *doff = nullptr;
    if ((rc = map_host(ctx, sink->entities, V * sink->capacity * 8, &de))) return rc;
    if ((rc = map_host(ctx, sink->offsets, V * 9 * 4, &doff))) return rc;
    if (!ctx->d_ent_counts) {
        const uint32_t chunks = visible_entity_chunks(ctx->cfg.max_entities);
        CU(dalloc(&ctx->d_ent_counts, V * chunks * 8));
        ctx->ent_chunks = chunks;
    }
    if ((rc = make_keys_resident(ctx))) return rc;
    ctx->ent_sink_d = reinterpret_cast<uint64_t *>(de); ctx->ent_off_d = doff; ctx->ent_cap = sink->capacity;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_column_sinks(b200vis_ctx *ctx, const b200vis_column_sinks *sinks) {
    CHECK_CTX_JOIN();
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->have_colsink = false;
    ctx->col_gt_d = nullptr; ctx->col_gt_bits_d = nullptr; ctx->col_vv_bits_d = nullptr; ctx->col_vv_d = nullptr;
    if (!sinks) return B200VIS_OK;
    if (sinks->global_transforms && sinks->gt_stride_floats != 12 && sinks->gt_stride_floats != 16)
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_column_sinks: gt_stride_floats must be 12 or 16");
    const size_t N = ctx->cfg.max_entities, W = (N + 31) / 32;
    int32_t rc;
    uint32_t *d = nullptr;
    if ((rc = map_host(ctx, sinks->global_transforms, N * sinks->gt_stride_floats * 4, &d))) return rc;
    ctx->col_gt_d = reinterpret_cast<float *>(d);
    if ((rc = map_host(ctx, sinks->gt_changed_bits, W * 4, &ctx->col_gt_bits_d))) return rc;
    if ((rc = map_host(ctx, sinks->view_visibility, N, &d))) return rc;
    ctx->col_vv_d = reinterpret_cast<uint8_t *>(d);
    if ((rc = map_host(ctx, sinks->vv_changed_bits, W * 4, &ctx->col_vv_bits_d))) return rc;
    if (!ctx->d_vv_shadow) CU(dalloc(&ctx->d_vv_shadow, N + 32));
    CU(cudaMemset(ctx->d_vv_shadow, 0xFF, N + 32));      // the host column's contents are unknown: the first write-back sends all
    ctx->colsink = *sinks;
    ctx->have_colsink = true;
    ctx->gt_aos_valid = false;
    return B200VIS_OK;
}
extern "C" int32_t b200vis_writeback_columns_ex(b200vis_ctx *ctx, uint32_t which);
extern "C" int32_t b200vis_writeback_columns(b200vis_ctx *ctx) { return b200vis_writeback_columns_ex(ctx, B200VIS_WB_GLOBAL_TRANSFORM | B200VIS_WB_VIEW_VISIBILITY); }
extern "C" int32_t b200vis_writeback_columns_ex(b200vis_ctx *ctx, uint32_t which) {
    CHECK_CTX();
    if (!ctx->have_colsink) return fail(ctx, B200VIS_ERR_NOT_READY, "writeback_columns: call b200vis_set_column_sinks first");
    // on the main stream, right behind the tile pass (and the shadow-culling stage, if the caller ran it): the tail of the
    // frame (list expansion, clusters) runs beside it on the side stream, the next frame's tile pass behind it
    const bool wgt = which & B200VIS_WB_GLOBAL_TRANSFORM, wvv = which & B200VIS_WB_VIEW_VISIBILITY;
    float *gt_sink = wgt ? ctx->col_gt_d : nullptr;
    static int dense_env = -1;
    if (dense_env < 0) { const char *e = getenv("B200VIS_WRITEBACK_DENSE"); dense_env = e ? atoi(e) : 1; }
    if (gt_sink && dense_env && (uint64_t)ctx->last_gt_changed * 2u >= ctx->n && ctx->n) {
        // most rows changed last frame (and will again): repack the whole column on the device (HBM speed) and let the copy
        // engine move it -- unchanged rows are rewritten with the bytes the host already holds.  Sparse frames take the
        // scatter kernel below instead (it touches only the changed rows).
        // (the staging copy starts as the device column in the host's layout, so that rows the scatter kernel skips -- unchanged
        // ones -- still carry the bytes the host holds)
        const uint32_t stride = ctx->colsink.gt_stride_floats;
        if (!ctx->d_gt_aos) { CU(dalloc(&ctx->d_gt_aos, (size_t)ctx->cfg.max_entities * 16)); ctx->gt_aos_valid = false; }
        if (!ctx->gt_aos_valid) { launch_pack_gt(ctx->stream, ctx->rows, 0, ctx->n, ctx->d_gt_aos, stride); ctx->gt_aos_valid = true; }
        // the same kernel as the sparse path (512-byte contiguous stores through shared memory), aimed at HBM instead of PCIe
        launch_writeback_columns(ctx->stream, ctx->rows, ctx->d_gt_aos, stride, wgt ? ctx->col_gt_bits_d : nullptr,
                                 wvv ? ctx->col_vv_d : nullptr, wvv ? ctx->col_vv_bits_d : nullptr, ctx->d_vv_shadow);
        CU(cudaMemcpyAsync(ctx->colsink.global_transforms, ctx->d_gt_aos, (size_t)ctx->n * stride * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaGetLastError());
        return B200VIS_OK;
    }
    if (gt_sink) ctx->gt_aos_valid = false;   // rows written straight to the host bypass the staging copy: it is stale from here on
    launch_writeback_columns(ctx->stream, ctx->rows, gt_sink, ctx->colsink.gt_stride_floats, wgt ? ctx->col_gt_bits_d : nullptr,
                             wvv ? ctx->col_vv_d : nullptr, wvv ? ctx->col_vv_bits_d : nullptr, ctx->d_vv_shadow);
    CU(cudaGetLastError());
    return B200VIS_OK;
}

// ---- write-back into the caller's archetype tables (b200vis_set_tables) ------------------------------------------------
// The host keeps the slot -> row maps of every table back to back exactly as the device holds them, plus the inverse
// row -> map entry it needs to validate calls and to apply moves.  Updates reach the device as (entry, row) pairs.
static constexpr uint32_t kUnmapped = B200VIS_UNMAPPED;

// Map updates are queued on the host and sent as one batch right before the device next reads the maps
// (b200vis_writeback_tables, b200vis_compact_topology, b200vis_set_tables), so b200vis_set_table_rows and the edits never
// wait for the stream.  A batch = the touched map entries with their host values at flush time + the shadow resets.
static void queue_table_updates(b200vis_ctx *ctx, const std::vector<uint32_t> &touched, const std::vector<uint32_t> &reset) {
    ctx->pend_touched.insert(ctx->pend_touched.end(), touched.begin(), touched.end());
    ctx->pend_reset.insert(ctx->pend_reset.end(), reset.begin(), reset.end());
}
static int32_t flush_table_updates(b200vis_ctx *ctx) {
    std::vector<uint32_t> &touched = ctx->pend_touched, &reset = ctx->pend_reset;
    if (touched.empty() && reset.empty()) return B200VIS_OK;
    std::sort(touched.begin(), touched.end());
    touched.erase(std::unique(touched.begin(), touched.end()), touched.end());
    const size_t n_set = touched.size(), n_reset = reset.size(), set_bytes = n_set * 8, bytes = set_bytes + n_reset * 4;
    if (ctx->ev_tab) CU(cudaEventSynchronize(ctx->ev_tab));   // the last batch's staging copy has been read
    else CU(cudaEventCreateWithFlags(&ctx->ev_tab, cudaEventDisableTiming));
    if (bytes > ctx->h_tab_stage_cap) {
        if (ctx->h_tab_stage) cudaFreeHost(ctx->h_tab_stage);
        ctx->h_tab_stage = nullptr; ctx->h_tab_stage_cap = 0;
        const size_t cap = std::max<size_t>(2 * bytes, 4096);
        CU(cudaMallocHost(&ctx->h_tab_stage, cap));
        ctx->h_tab_stage_cap = cap;
    }
    if (bytes > ctx->tab_upd_cap) {
        CU(cudaStreamSynchronize(ctx->stream));               // an earlier batch's kernel may still read the old buffer
        if (ctx->d_tab_upd) cudaFree(ctx->d_tab_upd);
        ctx->d_tab_upd = nullptr; ctx->tab_upd_cap = 0;
        CU(dalloc(&ctx->d_tab_upd, ctx->h_tab_stage_cap));
        ctx->tab_upd_cap = ctx->h_tab_stage_cap;
    }
    uint2 *set = reinterpret_cast<uint2 *>(ctx->h_tab_stage);
    for (size_t i = 0; i < n_set; ++i) set[i] = make_uint2(touched[i], ctx->h_tab_map[touched[i]]);
    if (n_reset) memcpy(ctx->h_tab_stage + set_bytes, reset.data(), n_reset * 4);
    CU(cudaMemcpyAsync(ctx->d_tab_upd, ctx->h_tab_stage, bytes, cudaMemcpyHostToDevice, ctx->stream));
    launch_update_table_map(ctx->stream, ctx->d_tab_map, reinterpret_cast<const uint2 *>(ctx->d_tab_upd), (uint32_t)n_set, ctx->d_tvv_shadow,
                            reinterpret_cast<const uint32_t *>(ctx->d_tab_upd + set_bytes), (uint32_t)n_reset, ctx->d_tab_fresh);
    CU(cudaGetLastError());
    CU(cudaEventRecord(ctx->ev_tab, ctx->stream));
    touched.clear(); reset.clear();
    return B200VIS_OK;
}

// b200vis_set_topology: every slot unmapped (the tables stay registered)
static int32_t tables_unmap_all(b200vis_ctx *ctx) {
    if (!ctx->tables_set) return B200VIS_OK;
    std::fill(ctx->h_tab_map.begin(), ctx->h_tab_map.end(), kUnmapped);
    std::fill(ctx->row_slot.begin(), ctx->row_slot.end(), kUnmapped);
    ctx->pend_touched.clear();                                // every entry is unmapped below
    if (!ctx->h_tab_map.empty()) CU(cudaMemsetAsync(ctx->d_tab_map, 0xFF, ctx->h_tab_map.size() * 4, ctx->stream));
    return B200VIS_OK;
}

// b200vis_edit_topology: the despawned rows leave their slots
static int32_t tables_unmap_rows(b200vis_ctx *ctx, uint32_t n_rows, const uint32_t *rows) {
    if (!ctx->tables_set) return B200VIS_OK;
    std::vector<uint32_t> touched;
    for (uint32_t i = 0; i < n_rows; ++i) {
        const uint32_t r = rows[i];
        if (r >= ctx->row_slot.size() || ctx->row_slot[r] == kUnmapped) continue;
        ctx->h_tab_map[ctx->row_slot[r]] = kUnmapped;
        touched.push_back(ctx->row_slot[r]);
        ctx->row_slot[r] = kUnmapped;
    }
    queue_table_updates(ctx, touched, {});
    return B200VIS_OK;
}

// b200vis_compact_topology, host side (the device maps are renumbered by the compaction's own kernels): every mapped row
// is live, so it survives
static void tables_renumber(b200vis_ctx *ctx, const std::vector<uint32_t> &old_to_new) {
    if (!ctx->tables_set) return;
    std::fill(ctx->row_slot.begin(), ctx->row_slot.end(), kUnmapped);
    for (size_t i = 0; i < ctx->h_tab_map.size(); ++i) {
        uint32_t &r = ctx->h_tab_map[i];
        if (r == kUnmapped) continue;
        r = old_to_new[r];
        ctx->row_slot[r] = (uint32_t)i;
    }
}

// ---- registrations of the caller's columns: page-rounded ranges, overlapping ones merged; stale ones released before new
// ones are made ----
using Range = std::pair<uintptr_t, uintptr_t>;
struct ColumnRanges { std::vector<Range> need, changed; };   // changed = memory that may have been reallocated

static Range page_range(const void *p, size_t bytes) {
    const uintptr_t page = (uintptr_t)sysconf(_SC_PAGESIZE), a = (uintptr_t)p;
    return Range{a & ~(page - 1), (a + bytes + page - 1) & ~(page - 1)};
}
template <typename Fn>
static void cull_columns(size_t cap, const b200vis_table_cull_inputs &cu, const b200vis_bounds_layout &bl, Fn &&fn) {
    fn(cu.aabbs, cap * bl.aabb_stride); fn(cu.aabb_changed_ticks, cap * 4);
    fn(cu.spheres, cap * bl.sphere_stride); fn(cu.sphere_changed_ticks, cap * 4);
    fn(cu.inherited_visibility, cap); fn(cu.iv_changed_ticks, cap * 4);
}
template <typename Fn>
static void range_columns(size_t cap, const b200vis_table_visibility_ranges &rg, uint32_t stride, Fn &&fn) {
    fn(rg.ranges, cap * stride); fn(rg.changed_ticks, cap * 4);
}
// every column of a table: the outputs, the Transform input, the cull inputs and the VisibilityRange column, as
// (pointer, bytes)
template <typename Fn>
static void table_columns(const b200vis_table &tb, const b200vis_table_inputs &in, uint32_t trs_stride, const b200vis_table_cull_inputs &cu,
                          const b200vis_bounds_layout &bl, const b200vis_table_visibility_ranges &rg, uint32_t range_stride, Fn &&fn) {
    const size_t cap = tb.capacity;
    fn(tb.global_transforms, cap * 64); fn(tb.gt_changed_ticks, cap * 4);
    fn(tb.view_visibility, cap); fn(tb.vv_changed_ticks, cap * 4);
    fn(in.transforms, cap * trs_stride); fn(in.transform_changed_ticks, cap * 4);
    cull_columns(cap, cu, bl, fn);
    range_columns(cap, rg, range_stride, fn);
}
// a column the registry uses: registered by the library unless its owner pinned it
static void need_column(b200vis_ctx *ctx, const void *p, size_t bytes, bool changed, ColumnRanges &cr) {
    if (!p || !bytes) return;
    if (changed) cr.changed.push_back(page_range(p, bytes));
    bool ours = false;
    for (const auto &r : ctx->host_regs) ours |= (uintptr_t)p >= r.first && (uintptr_t)p < r.first + r.second;
    void *d = nullptr;
    if (!ours && cudaHostGetDevicePointer(&d, const_cast<void *>(p), 0) == cudaSuccess) return;   // pinned by its owner
    cudaGetLastError();
    cr.need.push_back(page_range(p, bytes));
}
// A registered table as the kernels see it: the device aliases of its columns (NULL = not delivered).  The aliases are
// derived again whenever registrations may have moved.
static cudaError_t dev_table(const b200vis_table &tb, const b200vis_table_inputs &in, const b200vis_transform_layout &lay, uint32_t map_off,
                             uint32_t chunk_begin, DevTable &out) {
    void *alias[6] = {tb.global_transforms, tb.gt_changed_ticks, tb.view_visibility, tb.vv_changed_ticks,
                      const_cast<void *>(in.transforms), const_cast<uint32_t *>(in.transform_changed_ticks)};
    for (void *&p : alias) {
        if (!p || !tb.capacity) { p = nullptr; continue; }
        void *d = nullptr;
        const cudaError_t e = cudaHostGetDevicePointer(&d, p, 0);
        if (e != cudaSuccess) return e;
        p = d;
    }
    out = DevTable{static_cast<float4 *>(alias[0]), static_cast<uint32_t *>(alias[1]), static_cast<uint8_t *>(alias[2]),
                   static_cast<uint32_t *>(alias[3]), tb.len, map_off, chunk_begin, 0,
                   static_cast<const uint8_t *>(alias[4]), static_cast<const uint32_t *>(alias[5]),
                   lay.stride, lay.translation, lay.rotation, lay.scale};
    return cudaSuccess;
}

// Releases the registrations no range of cr.need is and those overlapping cr.changed, then registers what is missing.
// No table read or write-back may be in flight.  On failure every registration is released and the registry emptied.
static int32_t register_columns(b200vis_ctx *ctx, ColumnRanges &cr, const char *who) {
    std::sort(cr.need.begin(), cr.need.end());
    std::vector<Range> merged;
    for (const Range &r : cr.need) {
        if (!merged.empty() && r.first < merged.back().second) merged.back().second = std::max(merged.back().second, r.second);
        else merged.push_back(r);
    }
    std::vector<std::pair<uintptr_t, size_t>> regs;
    ctx->n_tab_chunks = 0;   // until the caller commits its registry, no write-back or read reaches a released range
    for (const auto &r : ctx->host_regs) {
        const uintptr_t lo = r.first, hi = r.first + r.second;
        bool stale = std::find(merged.begin(), merged.end(), Range{lo, hi}) == merged.end();
        for (const Range &c : cr.changed) stale |= c.first < hi && lo < c.second;
        if (stale) cudaHostUnregister(reinterpret_cast<void *>(lo));
        else regs.push_back(r);
    }
    cudaGetLastError();
    ctx->host_regs = regs;
    for (const Range &r : merged) {
        if (std::find(regs.begin(), regs.end(), std::make_pair(r.first, (size_t)(r.second - r.first))) != regs.end()) continue;
        const cudaError_t e = cudaHostRegister(reinterpret_cast<void *>(r.first), r.second - r.first, cudaHostRegisterMapped | cudaHostRegisterPortable);
        if (e != cudaSuccess) {
            cudaGetLastError();
            for (const auto &q : ctx->host_regs) cudaHostUnregister(reinterpret_cast<void *>(q.first));
            cudaGetLastError();
            ctx->host_regs.clear(); ctx->h_tabs.clear(); ctx->h_tab_in.clear(); ctx->tab_off.clear(); ctx->h_tab_map.clear();
            ctx->h_tab_cull.clear(); ctx->cull_attached = false;
            ctx->h_tab_caster.clear(); ctx->caster_attached = false;
            ctx->h_tab_range.clear(); ctx->range_attached = false;
            std::fill(ctx->row_slot.begin(), ctx->row_slot.end(), kUnmapped);
            ctx->n_tab_chunks = 0;
            return fail(ctx, B200VIS_ERR_CUDA, "%s: cudaHostRegister of %zu bytes at %p failed: %s", who, (size_t)(r.second - r.first),
                        reinterpret_cast<void *>(r.first), cudaGetErrorString(e));
        }
        ctx->host_regs.emplace_back(r.first, (size_t)(r.second - r.first));
    }
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_tables(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table *tables) {
    return b200vis_set_tables_ex(ctx, n_tables, tables, nullptr, nullptr);
}

extern "C" int32_t b200vis_set_tables_ex(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table *tables,
                                         const b200vis_table_inputs *inputs, const b200vis_transform_layout *layout) {
    CHECK_CTX_JOIN();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_tables: world_size > 1");
    if (n_tables && !tables) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: null tables");
    if (n_tables > B200VIS_MAX_TABLES) return fail(ctx, B200VIS_ERR_CAPACITY, "set_tables: %u tables > %u", n_tables, B200VIS_MAX_TABLES);
    const b200vis_table_inputs no_inputs{nullptr, nullptr};
    auto input = [&](uint32_t t) -> const b200vis_table_inputs & { return inputs ? inputs[t] : no_inputs; };
    uint64_t total = 0, chunks = 0;
    bool any_transforms = false;
    for (uint32_t t = 0; t < n_tables; ++t) {
        if (tables[t].len > tables[t].capacity)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: table %u has len %u > capacity %u", t, tables[t].len, tables[t].capacity);
        // the kernel stores float4 matrices and u32 ticks
        if ((uintptr_t)tables[t].global_transforms % 16u || (uintptr_t)tables[t].gt_changed_ticks % 4u || (uintptr_t)tables[t].vv_changed_ticks % 4u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: table %u: GlobalTransform needs 16-byte, tick columns 4-byte alignment", t);
        const b200vis_table_inputs &in = input(t);
        if ((in.transforms == nullptr) != (in.transform_changed_ticks == nullptr))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: table %u: transforms and transform_changed_ticks must both be NULL or both be set", t);
        // the kernel reads f32 fields and u32 ticks
        if ((uintptr_t)in.transforms % 4u || (uintptr_t)in.transform_changed_ticks % 4u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: table %u: input columns need 4-byte alignment", t);
        any_transforms |= in.transforms != nullptr;
        total += tables[t].capacity;
        chunks += (tables[t].len + 127u) / 128u;
    }
    if (any_transforms) {
        if (!layout) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: a table has transforms but no layout was given");
        const uint64_t lo[3] = {layout->translation, layout->rotation, layout->scale}, sz[3] = {12, 16, 12};
        if (layout->stride % 4u || lo[0] % 4u || lo[1] % 4u || lo[2] % 4u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: Transform layout fields and stride need 4-byte alignment");
        for (int i = 0; i < 3; ++i) {
            if (lo[i] + sz[i] > layout->stride)
                return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: Transform field at %llu runs past stride %u", (unsigned long long)lo[i], layout->stride);
            for (int j = 0; j < i; ++j)
                if (lo[i] < lo[j] + sz[j] && lo[j] < lo[i] + sz[i])
                    return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_tables: Transform fields at %llu and %llu overlap", (unsigned long long)lo[j], (unsigned long long)lo[i]);
        }
    }
    const b200vis_transform_layout lay = any_transforms ? *layout : b200vis_transform_layout{0, 0, 0, 0};
    if (total > (1ull << 31)) return fail(ctx, B200VIS_ERR_CAPACITY, "set_tables: %llu slots in all > 2^31", (unsigned long long)total);
    CU(cudaStreamSynchronize(ctx->stream));   // no write-back or read in flight reads the old registry or registrations
    { const int32_t frc = flush_table_updates(ctx); if (frc) return frc; }   // queued entries index the current layout
    const uint32_t n_old = (uint32_t)ctx->h_tabs.size();
    auto moved = [&](uint32_t t) {            // table t's memory is not what it was (or t is new or gone)
        if (t >= n_old || t >= n_tables) return true;
        const b200vis_table &a = ctx->h_tabs[t], &b = tables[t];
        const b200vis_table_inputs &ai = ctx->h_tab_in[t], &bi = input(t);
        return a.global_transforms != b.global_transforms || a.gt_changed_ticks != b.gt_changed_ticks ||
               a.view_visibility != b.view_visibility || a.vv_changed_ticks != b.vv_changed_ticks || a.capacity != b.capacity ||
               ai.transforms != bi.transforms || ai.transform_changed_ticks != bi.transform_changed_ticks ||
               (ai.transforms && ctx->tab_layout.stride != lay.stride);
    };
    // ---- the new maps: the entries below both capacities carry over ----
    std::vector<uint32_t> off(n_tables), map((size_t)total, kUnmapped), reset;
    bool same_layout = ctx->tables_set && n_tables == n_old;
    for (uint32_t t = 0, o = 0; t < n_tables; o += tables[t].capacity, ++t) {
        off[t] = o;
        if (t >= n_old) continue;
        const uint32_t keep = std::min(tables[t].capacity, ctx->h_tabs[t].capacity);
        same_layout &= tables[t].capacity == ctx->h_tabs[t].capacity;
        std::copy_n(ctx->h_tab_map.begin() + ctx->tab_off[t], keep, map.begin() + o);
        if (tables[t].view_visibility != ctx->h_tabs[t].view_visibility)   // a new column: its bytes are sent again
            for (uint32_t s = 0; s < keep; ++s) if (map[o + s] != kUnmapped) reset.push_back(map[o + s]);
    }
    // ---- registrations: every current column, plus the cull inputs of tables that stay (kept until they are attached
    // again); the columns of moved tables, old and new, are memory that may have been reallocated ----
    const b200vis_table_cull_inputs no_cull{};
    auto kept_cull = [&](uint32_t t) -> const b200vis_table_cull_inputs & {
        return t < n_old && t < ctx->h_tab_cull.size() && !moved(t) ? ctx->h_tab_cull[t] : no_cull;
    };
    const b200vis_table_visibility_ranges no_range{};
    auto held_range = [&](uint32_t t) -> const b200vis_table_visibility_ranges & {
        return t < ctx->h_tab_range.size() ? ctx->h_tab_range[t] : no_range;
    };
    std::vector<b200vis_table_visibility_ranges> kept_range(n_tables);
    for (uint32_t t = 0; t < n_tables; ++t) if (t < n_old && !moved(t)) kept_range[t] = held_range(t);
    ColumnRanges cr;
    for (uint32_t t = 0; t < n_tables; ++t)
        table_columns(tables[t], input(t), lay.stride, kept_cull(t), ctx->cull_layout, kept_range[t], ctx->range_layout.stride,
                      [&](const void *p, size_t bytes) { need_column(ctx, p, bytes, moved(t), cr); });
    for (uint32_t t = 0; t < n_old; ++t)
        if (moved(t))
            table_columns(ctx->h_tabs[t], ctx->h_tab_in[t], ctx->tab_layout.stride, t < ctx->h_tab_cull.size() ? ctx->h_tab_cull[t] : no_cull,
                          ctx->cull_layout, held_range(t), ctx->range_layout.stride,
                          [&](const void *p, size_t bytes) { if (p && bytes) cr.changed.push_back(page_range(p, bytes)); });
    { const int32_t rrc = register_columns(ctx, cr, "set_tables"); if (rrc) return rrc; }
    // ---- the device registry: table descriptors, chunk -> table, and the maps when their layout changed ----
    std::vector<DevTable> dt(n_tables);
    std::vector<uint32_t> chunk_table((size_t)chunks);
    for (uint32_t t = 0, c = 0; t < n_tables; ++t) {
        CU(dev_table(tables[t], input(t), lay, off[t], c, dt[t]));
        for (uint32_t k = 0; k < (tables[t].len + 127u) / 128u; ++k) chunk_table[c++] = t;
    }
    const size_t N = ctx->cfg.max_entities;
    if (!ctx->d_tabs) CU(dalloc(&ctx->d_tabs, B200VIS_MAX_TABLES));
    if (!ctx->d_tab_total) CU(dalloc(&ctx->d_tab_total, 1));
    if (!ctx->d_tvv_shadow) { CU(dalloc(&ctx->d_tvv_shadow, N + 32)); CU(cudaMemset(ctx->d_tvv_shadow, 0xFF, N + 32)); }
    if (chunks > ctx->tab_chunks_cap) {
        if (ctx->d_tab_chunks) cudaFree(ctx->d_tab_chunks);
        ctx->d_tab_chunks = nullptr; ctx->tab_chunks_cap = 0;
        CU(dalloc(&ctx->d_tab_chunks, (size_t)chunks));
        ctx->tab_chunks_cap = (uint32_t)chunks;
    }
    if (total > ctx->tab_map_cap) {
        if (ctx->d_tab_map) cudaFree(ctx->d_tab_map);
        ctx->d_tab_map = nullptr; ctx->tab_map_cap = 0;
        CU(dalloc(&ctx->d_tab_map, (size_t)total));
        ctx->tab_map_cap = (size_t)total;
    }
    cudaStream_t st = ctx->stream;
    const uint32_t total32 = (uint32_t)total;
    if (n_tables) CU(cudaMemcpyAsync(ctx->d_tabs, dt.data(), dt.size() * sizeof(DevTable), cudaMemcpyHostToDevice, st));
    if (chunks) CU(cudaMemcpyAsync(ctx->d_tab_chunks, chunk_table.data(), (size_t)chunks * 4, cudaMemcpyHostToDevice, st));
    if (!same_layout && total) CU(cudaMemcpyAsync(ctx->d_tab_map, map.data(), (size_t)total * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(ctx->d_tab_total, &total32, 4, cudaMemcpyHostToDevice, st));
    uint8_t *old_fresh = nullptr;
    if (!same_layout || !ctx->d_tab_fresh) {
        // the "read in full" marks move with the map entries that carry over (the cull inputs of a table that stays
        // are attached again without a full read)
        old_fresh = ctx->d_tab_fresh; ctx->d_tab_fresh = nullptr;
        CU(dalloc(&ctx->d_tab_fresh, std::max<size_t>(ctx->tab_map_cap, 1)));
        for (uint32_t t = 0; old_fresh && t < std::min(n_old, n_tables); ++t) {
            const uint32_t keep = std::min(tables[t].capacity, ctx->h_tabs[t].capacity);
            if (keep) CU(cudaMemcpyAsync(ctx->d_tab_fresh + off[t], old_fresh + ctx->tab_off[t], keep, cudaMemcpyDeviceToDevice, st));
        }
    }
    CU(cudaStreamSynchronize(st));
    if (old_fresh) cudaFree(old_fresh);
    // ---- commit ----
    // slots that come below len may hold "read in full" marks a cull read skipped while they were past it
    for (uint32_t t = 0; t < n_tables; ++t) ctx->cull_fresh_pending |= tables[t].len > (t < n_old ? ctx->h_tabs[t].len : 0u);
    ctx->h_tabs.assign(tables, tables + n_tables);
    ctx->h_tab_in.resize(n_tables);
    for (uint32_t t = 0; t < n_tables; ++t) ctx->h_tab_in[t] = input(t);
    ctx->tab_layout = lay;
    ctx->tab_off = std::move(off);
    ctx->h_tab_map = std::move(map);
    ctx->row_slot.assign(N, kUnmapped);
    for (size_t i = 0; i < ctx->h_tab_map.size(); ++i) if (ctx->h_tab_map[i] != kUnmapped) ctx->row_slot[ctx->h_tab_map[i]] = (uint32_t)i;
    ctx->n_tab_chunks = (uint32_t)chunks;
    ctx->tables_set = true;
    ctx->cull_attached = false;              // the cull inputs are attached again by b200vis_set_table_cull_inputs
    ctx->caster_attached = false; ctx->h_tab_caster.clear();   // ... and the table casters by b200vis_set_table_shadow_casters
    ctx->range_attached = false; ctx->h_tab_range = std::move(kept_range);   // ... and the ranges (kept: registrations held)
    queue_table_updates(ctx, {}, reset);
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_table_rows(b200vis_ctx *ctx, uint32_t table, uint32_t first_slot, uint32_t count, const uint32_t *rows) {
    CHECK_CTX();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_table_rows: world_size > 1");
    if (table >= ctx->h_tabs.size()) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_rows: table %u of %zu", table, ctx->h_tabs.size());
    if ((uint64_t)first_slot + count > ctx->h_tabs[table].capacity)
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_rows: slots [%u, %llu) past table %u's capacity %u", first_slot,
                    (unsigned long long)first_slot + count, table, ctx->h_tabs[table].capacity);
    if (count && !rows) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_rows: null rows");
    const Plan *hp = ctx->topology_set ? ctx->hplan : nullptr;
    for (uint32_t i = 0; i < count; ++i) {
        const uint32_t r = rows[i];
        if (r != kUnmapped && (!hp || r >= ctx->n || !hp->alive[r]))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_rows: row %u (slot %u) is out of range or despawned", r, first_slot + i);
    }
    std::vector<uint32_t> touched, reset;
    const uint32_t base = ctx->tab_off[table] + first_slot;
    for (uint32_t i = 0; i < count; ++i) {
        const uint32_t e = base + i, r = rows[i], old = ctx->h_tab_map[e];
        if (old == r) continue;
        if (old != kUnmapped) ctx->row_slot[old] = kUnmapped;
        if (r != kUnmapped) {
            const uint32_t prev = ctx->row_slot[r];
            if (prev != kUnmapped) { ctx->h_tab_map[prev] = kUnmapped; touched.push_back(prev); }
            ctx->row_slot[r] = e;
            reset.push_back(r);          // a new slot: what it holds is unknown
        }
        ctx->h_tab_map[e] = r;
        touched.push_back(e);
    }
    ctx->cull_fresh_pending |= !touched.empty();
    queue_table_updates(ctx, touched, reset);
    return B200VIS_OK;
}

static bool cull_reads(const b200vis_table_cull_inputs &c) {
    return c.aabbs || c.spheres || c.inherited_visibility || c.flags;
}
// the same columns, flags and used layout fields: the table needs no full read
static bool cull_same(const b200vis_table_cull_inputs &a, const b200vis_bounds_layout &la, const b200vis_table_cull_inputs &b,
                      const b200vis_bounds_layout &lb) {
    return a.aabbs == b.aabbs && a.aabb_changed_ticks == b.aabb_changed_ticks && a.spheres == b.spheres &&
           a.sphere_changed_ticks == b.sphere_changed_ticks && a.inherited_visibility == b.inherited_visibility &&
           a.iv_changed_ticks == b.iv_changed_ticks && a.flags == b.flags &&
           (!a.aabbs || (la.aabb_stride == lb.aabb_stride && la.aabb_center == lb.aabb_center && la.aabb_half_extents == lb.aabb_half_extents)) &&
           (!a.spheres || a.aabbs || (la.sphere_stride == lb.sphere_stride && la.sphere_center == lb.sphere_center && la.sphere_radius == lb.sphere_radius));
}

// table t's cull inputs as k_read_table_cull sees them (the aliases derived from the current registrations)
static cudaError_t dev_cull(const b200vis_ctx *ctx, uint32_t t, const b200vis_table_cull_inputs &c, const b200vis_bounds_layout &lay,
                            DevTableCull &d) {
    const uint32_t cap = ctx->h_tabs[t].capacity;
    cudaError_t lost = cudaSuccess;
    auto alias = [&](const void *p) -> const void * {
        void *dp = nullptr;
        if (!p || !cap) return nullptr;
        const cudaError_t e = cudaHostGetDevicePointer(&dp, const_cast<void *>(p), 0);
        if (e != cudaSuccess) lost = e;
        return dp;
    };
    const bool aabb = c.aabbs != nullptr;
    d = DevTableCull{};
    d.bnd = static_cast<const uint8_t *>(alias(aabb ? c.aabbs : c.spheres));
    d.bnd_ticks = static_cast<const uint32_t *>(alias(aabb ? c.aabb_changed_ticks : c.sphere_changed_ticks));
    d.iv = static_cast<const uint8_t *>(alias(c.inherited_visibility));
    d.iv_ticks = static_cast<const uint32_t *>(alias(c.iv_changed_ticks));
    d.flags = c.flags | (aabb ? B200VIS_F_HAS_AABB : c.spheres ? B200VIS_F_HAS_SPHERE : 0u);
    d.read = cull_reads(c) && cap ? 1u : 0u;
    d.stride = aabb ? lay.aabb_stride : lay.sphere_stride;
    d.c_off = aabb ? lay.aabb_center : lay.sphere_center;
    d.e_off = aabb ? lay.aabb_half_extents : lay.sphere_radius;
    d.is_aabb = aabb;
    return lost;
}
static const b200vis_table_visibility_ranges &held_range(const b200vis_ctx *ctx, uint32_t t) {
    static const b200vis_table_visibility_ranges none{};
    return t < ctx->h_tab_range.size() ? ctx->h_tab_range[t] : none;
}
// the device form of per-table range entries: the aliases of the registered columns, derived again whenever
// registrations may have moved
static cudaError_t dev_ranges(const b200vis_ctx *ctx, const std::vector<b200vis_table_visibility_ranges> &rg, std::vector<DevTableRange> &out) {
    out.assign(rg.size(), DevTableRange{nullptr, nullptr});
    for (size_t t = 0; t < rg.size(); ++t) {
        if (!rg[t].ranges || !ctx->h_tabs[t].capacity) continue;
        void *d = nullptr, *dt = nullptr;
        cudaError_t e = cudaHostGetDevicePointer(&d, const_cast<void *>(rg[t].ranges), 0);
        if (e == cudaSuccess) e = cudaHostGetDevicePointer(&dt, const_cast<uint32_t *>(rg[t].changed_ticks), 0);
        if (e != cudaSuccess) return e;
        out[t] = DevTableRange{static_cast<const uint8_t *>(d), static_cast<const uint32_t *>(dt)};
    }
    return cudaSuccess;
}

extern "C" int32_t b200vis_set_table_cull_inputs(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table_cull_inputs *inputs,
                                                 const b200vis_bounds_layout *layout) {
    CHECK_CTX_JOIN();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_table_cull_inputs: world_size > 1");
    if (!ctx->tables_set || ctx->h_tabs.empty()) return fail(ctx, B200VIS_ERR_NOT_READY, "set_table_cull_inputs: no tables are registered");
    if (n_tables != ctx->h_tabs.size())
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: %u entries for %zu registered tables", n_tables, ctx->h_tabs.size());
    if (!inputs) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: null inputs");
    constexpr uint32_t kArchetypeBits = B200VIS_F_NO_FRUSTUM_CULLING | B200VIS_F_HAS_VIS_RANGE | B200VIS_F_NO_CPU_CULLING | B200VIS_F_SPHERE_FROM_GT;
    bool any_aabb = false, any_sphere = false;
    for (uint32_t t = 0; t < n_tables; ++t) {
        const b200vis_table_cull_inputs &c = inputs[t];
        if ((c.aabbs == nullptr) != (c.aabb_changed_ticks == nullptr) || (c.spheres == nullptr) != (c.sphere_changed_ticks == nullptr) ||
            (c.inherited_visibility == nullptr) != (c.iv_changed_ticks == nullptr))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: table %u: a column and its ticks must both be NULL or both be set", t);
        // the kernel reads f32 fields and u32 ticks
        if ((uintptr_t)c.aabbs % 4u || (uintptr_t)c.spheres % 4u || (uintptr_t)c.aabb_changed_ticks % 4u ||
            (uintptr_t)c.sphere_changed_ticks % 4u || (uintptr_t)c.iv_changed_ticks % 4u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: table %u: columns need 4-byte alignment", t);
        if (c.flags & ~kArchetypeBits)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: table %u: flags 0x%x has bits other than the per-archetype ones", t, c.flags);
        any_aabb |= c.aabbs != nullptr; any_sphere |= c.spheres != nullptr;
        // while ranges are attached, HAS_VIS_RANGE and a range column go together (b200vis_set_table_visibility_ranges)
        if (ctx->range_attached && ((c.flags & B200VIS_F_HAS_VIS_RANGE) != 0) != (ctx->h_tab_range[t].ranges != nullptr))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: table %u: HAS_VIS_RANGE %s while its VisibilityRange "
                        "column is %s; detach the ranges first", t, (c.flags & B200VIS_F_HAS_VIS_RANGE) ? "set" : "clear",
                        ctx->h_tab_range[t].ranges ? "attached" : "absent");
    }
    if ((any_aabb || any_sphere) && !layout)
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: a table has aabbs or spheres but no layout was given");
    auto check_struct = [&](const char *name, uint32_t stride, const uint64_t (&lo)[2], const uint64_t (&sz)[2]) -> int32_t {
        if (stride % 4u || lo[0] % 4u || lo[1] % 4u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: %s layout fields and stride need 4-byte alignment", name);
        for (int i = 0; i < 2; ++i)
            if (lo[i] + sz[i] > stride)
                return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: %s field at %llu runs past stride %u", name, (unsigned long long)lo[i], stride);
        if (lo[0] < lo[1] + sz[1] && lo[1] < lo[0] + sz[0])
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_cull_inputs: %s fields at %llu and %llu overlap", name,
                        (unsigned long long)lo[0], (unsigned long long)lo[1]);
        return B200VIS_OK;
    };
    if (any_aabb) {
        const int32_t rc = check_struct("Aabb", layout->aabb_stride, {layout->aabb_center, layout->aabb_half_extents}, {12, 12});
        if (rc) return rc;
    }
    if (any_sphere) {
        const int32_t rc = check_struct("Sphere", layout->sphere_stride, {layout->sphere_center, layout->sphere_radius}, {12, 4});
        if (rc) return rc;
    }
    b200vis_bounds_layout lay{};
    if (any_aabb) { lay.aabb_stride = layout->aabb_stride; lay.aabb_center = layout->aabb_center; lay.aabb_half_extents = layout->aabb_half_extents; }
    if (any_sphere) { lay.sphere_stride = layout->sphere_stride; lay.sphere_center = layout->sphere_center; lay.sphere_radius = layout->sphere_radius; }
    CU(cudaStreamSynchronize(ctx->stream));   // no read in flight reads the old cull columns or registrations
    const b200vis_table_cull_inputs none{};
    auto prev = [&](uint32_t t) -> const b200vis_table_cull_inputs & { return t < ctx->h_tab_cull.size() ? ctx->h_tab_cull[t] : none; };
    std::vector<bool> full(n_tables);
    for (uint32_t t = 0; t < n_tables; ++t) full[t] = cull_reads(inputs[t]) && !cull_same(inputs[t], lay, prev(t), ctx->cull_layout);
    // ---- registrations: every table's columns with the new cull inputs; cull columns that changed may be reallocated ----
    const uint32_t chunks = ctx->n_tab_chunks;
    ColumnRanges cr;
    for (uint32_t t = 0; t < n_tables; ++t) {
        const bool moved = !cull_same(inputs[t], lay, prev(t), ctx->cull_layout);
        table_columns(ctx->h_tabs[t], ctx->h_tab_in[t], ctx->tab_layout.stride, inputs[t], lay, held_range(ctx, t), ctx->range_layout.stride,
                      [&](const void *p, size_t bytes) { need_column(ctx, p, bytes, false, cr); });
        if (moved) {
            auto changed = [&](const void *p, size_t bytes) { if (p && bytes) cr.changed.push_back(page_range(p, bytes)); };
            cull_columns(ctx->h_tabs[t].capacity, inputs[t], lay, changed);
            cull_columns(ctx->h_tabs[t].capacity, prev(t), ctx->cull_layout, changed);
        }
    }
    { const int32_t rrc = register_columns(ctx, cr, "set_table_cull_inputs"); if (rrc) return rrc; }
    ctx->n_tab_chunks = chunks;
    // From here on registrations may have moved: a failure detaches the cull inputs (nothing reads them until the next
    // call, which reads every table it attaches in full) instead of leaving the device pointed at released ranges.
    auto detach = [&](cudaError_t e, const char *what, uint32_t t) {
        ctx->cull_attached = false;
        ctx->h_tab_cull.clear();
        ctx->range_attached = false; ctx->h_tab_range.clear();   // the ranges' aliases may have moved as well
        return fail(ctx, e == cudaErrorMemoryAllocation ? B200VIS_ERR_OUT_OF_MEMORY : B200VIS_ERR_CUDA,
                    "set_table_cull_inputs: table %u: %s: %s", t, what, cudaGetErrorString(e));
    };
    // ---- the registry's descriptors again: an output or Transform column sharing a page with a cull column may have
    // been registered anew, and its device alias is derived from the registration ----
    std::vector<DevTable> dt(n_tables);
    for (uint32_t t = 0, c = 0; t < n_tables; ++t) {
        const cudaError_t e = dev_table(ctx->h_tabs[t], ctx->h_tab_in[t], ctx->tab_layout, ctx->tab_off[t], c, dt[t]);
        if (e != cudaSuccess) return detach(e, "no device alias for a registered column", t);
        c += (ctx->h_tabs[t].len + 127u) / 128u;
    }
    // ---- the device form of the cull inputs, and the full-read marks of the tables attached anew ----
    std::vector<DevTableCull> dc(n_tables);
    bool any = false;
    for (uint32_t t = 0; t < n_tables; ++t) {
        const cudaError_t lost = dev_cull(ctx, t, inputs[t], lay, dc[t]);
        if (lost != cudaSuccess) return detach(lost, "no device alias for a registered column", t);
        any |= dc[t].read != 0;
    }
    cudaStream_t st = ctx->stream;
    cudaError_t e = cudaSuccess;
    if (!ctx->d_tab_cull && (e = dalloc(&ctx->d_tab_cull, B200VIS_MAX_TABLES)) != cudaSuccess) return detach(e, "cudaMalloc", 0);
    if ((e = cudaMemcpyAsync(ctx->d_tabs, dt.data(), dt.size() * sizeof(DevTable), cudaMemcpyHostToDevice, st)) != cudaSuccess)
        return detach(e, "table descriptors", 0);
    if ((e = cudaMemcpyAsync(ctx->d_tab_cull, dc.data(), dc.size() * sizeof(DevTableCull), cudaMemcpyHostToDevice, st)) != cudaSuccess)
        return detach(e, "cull descriptors", 0);
    if (ctx->range_attached) {                  // a range column sharing a page with a cull column may have been registered anew
        std::vector<DevTableRange> dr;
        if ((e = dev_ranges(ctx, ctx->h_tab_range, dr)) != cudaSuccess) return detach(e, "no device alias for a range column", 0);
        if ((e = cudaMemcpyAsync(ctx->d_tab_range, dr.data(), dr.size() * sizeof(DevTableRange), cudaMemcpyHostToDevice, st)) != cudaSuccess)
            return detach(e, "range descriptors", 0);
    }
    bool pending = false;
    for (uint32_t t = 0; t < n_tables; ++t)
        if (full[t] && ctx->h_tabs[t].capacity) {
            if ((e = cudaMemsetAsync(ctx->d_tab_fresh + ctx->tab_off[t], 1, ctx->h_tabs[t].capacity, st)) != cudaSuccess)
                return detach(e, "full-read marks", t);
            pending = true;
        }
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return detach(e, "cudaStreamSynchronize", 0);
    // ---- commit ----
    ctx->cull_fresh_pending |= pending;
    ctx->h_tab_cull.assign(inputs, inputs + n_tables);
    ctx->cull_layout = lay;
    ctx->cull_attached = any;
    return B200VIS_OK;
}

extern "C" int32_t b200vis_set_table_shadow_casters(b200vis_ctx *ctx, uint32_t n_tables, const uint8_t *is_caster) {
    CHECK_CTX_JOIN();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_table_shadow_casters: world_size > 1");
    if (!n_tables && !is_caster) { ctx->caster_attached = false; ctx->h_tab_caster.clear(); return B200VIS_OK; }
    if (!ctx->tables_set || ctx->h_tabs.empty()) return fail(ctx, B200VIS_ERR_NOT_READY, "set_table_shadow_casters: no tables are registered");
    if (n_tables != ctx->h_tabs.size())
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_shadow_casters: %u entries for %zu registered tables", n_tables, ctx->h_tabs.size());
    if (!is_caster) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_shadow_casters: null is_caster");
    std::vector<uint8_t> bytes(n_tables);
    for (uint32_t t = 0; t < n_tables; ++t) bytes[t] = is_caster[t] ? 1u : 0u;
    if (!ctx->d_caster) CU(dalloc(&ctx->d_caster, ctx->cfg.max_entities));
    // the shadow stage reads each view's VisibleEntities as the visible-diff sets (as for b200vis_upload_shadow_casters)
    if (!ctx->diff_on) { const int32_t rc = b200vis_enable_visible_diff(ctx, 1); if (rc) return rc; }
    if (!ctx->d_tab_caster) CU(dalloc(&ctx->d_tab_caster, B200VIS_MAX_TABLES));
    cudaStream_t st = ctx->stream;
    CU(cudaStreamSynchronize(st));              // no read in flight reads the old bytes
    // a table whose byte changed (every table, on an attach after none) is read in full: the same mark as a changed cull
    // input, cleared by the read
    bool pending = false;
    for (uint32_t t = 0; t < n_tables; ++t) {
        const bool same = ctx->caster_attached && t < ctx->h_tab_caster.size() && ctx->h_tab_caster[t] == bytes[t];
        if (same || !ctx->h_tabs[t].capacity) continue;
        CU(cudaMemsetAsync(ctx->d_tab_fresh + ctx->tab_off[t], 1, ctx->h_tabs[t].capacity, st));
        pending = true;
    }
    CU(cudaMemcpyAsync(ctx->d_tab_caster, bytes.data(), n_tables, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    ctx->cull_fresh_pending |= pending;
    ctx->h_tab_caster = std::move(bytes);
    ctx->caster_attached = true;
    return B200VIS_OK;
}

static bool range_same(const b200vis_table_visibility_ranges &a, const b200vis_visibility_range_layout &la,
                       const b200vis_table_visibility_ranges &b, const b200vis_visibility_range_layout &lb) {
    return a.ranges == b.ranges && a.changed_ticks == b.changed_ticks &&
           (!a.ranges || (la.stride == lb.stride && la.start == lb.start && la.end == lb.end && la.use_aabb == lb.use_aabb));
}

extern "C" int32_t b200vis_set_table_visibility_ranges(b200vis_ctx *ctx, uint32_t n_tables, const b200vis_table_visibility_ranges *ranges,
                                                       const b200vis_visibility_range_layout *layout) {
    CHECK_CTX_JOIN();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "set_table_visibility_ranges: world_size > 1");
    if (!n_tables && !ranges) { ctx->range_attached = false; ctx->h_tab_range.clear(); return B200VIS_OK; }
    if (!ctx->tables_set || ctx->h_tabs.empty()) return fail(ctx, B200VIS_ERR_NOT_READY, "set_table_visibility_ranges: no tables are registered");
    if (n_tables != ctx->h_tabs.size())
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: %u entries for %zu registered tables", n_tables, ctx->h_tabs.size());
    if (!ranges) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: null ranges");
    bool any = false;
    for (uint32_t t = 0; t < n_tables; ++t) {
        const b200vis_table_visibility_ranges &r = ranges[t];
        if ((r.ranges == nullptr) != (r.changed_ticks == nullptr))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: table %u: ranges and changed_ticks must both be NULL or both be set", t);
        if ((uintptr_t)r.ranges % 4u || (uintptr_t)r.changed_ticks % 4u)   // the kernel reads f32 fields and u32 ticks
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: table %u: columns need 4-byte alignment", t);
        // no row is range-tested with parameters nobody supplied: HAS_VIS_RANGE in the attached cull inputs exactly when
        // the table has a range column
        const bool ranged = ctx->cull_attached && t < ctx->h_tab_cull.size() && (ctx->h_tab_cull[t].flags & B200VIS_F_HAS_VIS_RANGE);
        if (ranged != (r.ranges != nullptr))
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: table %u: %s, but its attached cull inputs %s HAS_VIS_RANGE", t,
                        r.ranges ? "a VisibilityRange column" : "no VisibilityRange column", ranged ? "carry" : "lack");
        any |= r.ranges != nullptr;
    }
    if (any && !layout) return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: a table has ranges but no layout was given");
    b200vis_visibility_range_layout lay{};
    if (any) {
        lay = *layout;
        const uint64_t lo[3] = {lay.start, lay.end, lay.use_aabb}, sz[3] = {4, 4, 1};
        if (lay.stride % 4u || lay.start % 4u || lay.end % 4u)
            return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: the float fields and the stride need 4-byte alignment");
        for (int i = 0; i < 3; ++i) {
            if (lo[i] + sz[i] > lay.stride)
                return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: field at %llu runs past stride %u", (unsigned long long)lo[i], lay.stride);
            for (int j = 0; j < i; ++j)
                if (lo[i] < lo[j] + sz[j] && lo[j] < lo[i] + sz[i])
                    return fail(ctx, B200VIS_ERR_INVALID_ARG, "set_table_visibility_ranges: fields at %llu and %llu overlap",
                                (unsigned long long)lo[j], (unsigned long long)lo[i]);
        }
    }
    // the resident range columns, as b200vis_upload_visibility_ranges allocates them
    if (!ctx->d_range_se) {
        CU(dalloc(&ctx->d_range_se, ctx->cfg.max_entities));
        CU(dalloc(&ctx->d_range_ua, ctx->cfg.max_entities));
        CU(dalloc(&ctx->d_range_views, 32));
    }
    if (!ctx->d_tab_range) CU(dalloc(&ctx->d_tab_range, B200VIS_MAX_TABLES));
    CU(cudaStreamSynchronize(ctx->stream));   // no read in flight reads the old range columns or registrations
    // a table whose entry changed is read in full: every table with ranges on an attach after none (h_tab_range is
    // empty then); b200vis_set_tables keeps the entries of the tables that stay, as for the cull inputs
    std::vector<bool> full(n_tables);
    for (uint32_t t = 0; t < n_tables; ++t)
        full[t] = ranges[t].ranges && (ctx->h_tab_range.empty() || !range_same(ranges[t], lay, held_range(ctx, t), ctx->range_layout));
    // ---- registrations: every table's columns with the new ranges; range columns that changed may be reallocated ----
    const b200vis_table_cull_inputs no_cull{};
    const uint32_t chunks = ctx->n_tab_chunks;
    ColumnRanges cr;
    for (uint32_t t = 0; t < n_tables; ++t) {
        const b200vis_table_cull_inputs &cu = t < ctx->h_tab_cull.size() ? ctx->h_tab_cull[t] : no_cull;
        table_columns(ctx->h_tabs[t], ctx->h_tab_in[t], ctx->tab_layout.stride, cu, ctx->cull_layout, ranges[t], lay.stride,
                      [&](const void *p, size_t bytes) { need_column(ctx, p, bytes, false, cr); });
        if (!range_same(ranges[t], lay, held_range(ctx, t), ctx->range_layout)) {
            auto changed = [&](const void *p, size_t bytes) { if (p && bytes) cr.changed.push_back(page_range(p, bytes)); };
            range_columns(ctx->h_tabs[t].capacity, ranges[t], lay.stride, changed);
            range_columns(ctx->h_tabs[t].capacity, held_range(ctx, t), ctx->range_layout.stride, changed);
        }
    }
    { const int32_t rrc = register_columns(ctx, cr, "set_table_visibility_ranges"); if (rrc) return rrc; }
    ctx->n_tab_chunks = chunks;
    // From here on registrations may have moved: a failure detaches the cull inputs and the ranges (the next calls read
    // every table they attach in full) instead of leaving the device pointed at released ranges.
    auto detach = [&](cudaError_t e, const char *what) {
        ctx->cull_attached = false; ctx->h_tab_cull.clear();
        ctx->range_attached = false; ctx->h_tab_range.clear();
        return fail(ctx, e == cudaErrorMemoryAllocation ? B200VIS_ERR_OUT_OF_MEMORY : B200VIS_ERR_CUDA,
                    "set_table_visibility_ranges: %s: %s", what, cudaGetErrorString(e));
    };
    // ---- the descriptors again: the table's, its cull inputs' and the ranges' aliases ----
    cudaStream_t st = ctx->stream;
    cudaError_t e = cudaSuccess;
    std::vector<DevTable> dt(n_tables);
    for (uint32_t t = 0, c = 0; t < n_tables; ++t) {
        if ((e = dev_table(ctx->h_tabs[t], ctx->h_tab_in[t], ctx->tab_layout, ctx->tab_off[t], c, dt[t])) != cudaSuccess)
            return detach(e, "no device alias for a registered column");
        c += (ctx->h_tabs[t].len + 127u) / 128u;
    }
    if ((e = cudaMemcpyAsync(ctx->d_tabs, dt.data(), dt.size() * sizeof(DevTable), cudaMemcpyHostToDevice, st)) != cudaSuccess)
        return detach(e, "table descriptors");
    if (ctx->cull_attached) {
        std::vector<DevTableCull> dc(n_tables);
        for (uint32_t t = 0; t < n_tables; ++t) if ((e = dev_cull(ctx, t, ctx->h_tab_cull[t], ctx->cull_layout, dc[t])) != cudaSuccess)
            return detach(e, "no device alias for a cull column");
        if ((e = cudaMemcpyAsync(ctx->d_tab_cull, dc.data(), dc.size() * sizeof(DevTableCull), cudaMemcpyHostToDevice, st)) != cudaSuccess)
            return detach(e, "cull descriptors");
    }
    std::vector<b200vis_table_visibility_ranges> rg(ranges, ranges + n_tables);
    std::vector<DevTableRange> dr;
    if ((e = dev_ranges(ctx, rg, dr)) != cudaSuccess) return detach(e, "no device alias for a range column");
    if ((e = cudaMemcpyAsync(ctx->d_tab_range, dr.data(), dr.size() * sizeof(DevTableRange), cudaMemcpyHostToDevice, st)) != cudaSuccess)
        return detach(e, "range descriptors");
    bool pending = false;
    for (uint32_t t = 0; t < n_tables; ++t)
        if (full[t] && ctx->h_tabs[t].capacity) {
            if ((e = cudaMemsetAsync(ctx->d_tab_fresh + ctx->tab_off[t], 1, ctx->h_tabs[t].capacity, st)) != cudaSuccess)
                return detach(e, "full-read marks");
            pending = true;
        }
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return detach(e, "cudaStreamSynchronize");
    // ---- commit ----
    ctx->cull_fresh_pending |= pending;
    ctx->h_tab_range = std::move(rg);
    ctx->range_layout = lay;
    ctx->range_attached = any;
    ctx->have_range = true;   // as after b200vis_upload_visibility_ranges: the cull kernels take the non-SIMPLE path
    return B200VIS_OK;
}

extern "C" int32_t b200vis_writeback_tables(b200vis_ctx *ctx, uint32_t which, uint32_t gt_tick, uint32_t vv_tick) {
    CHECK_CTX();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "writeback_tables: world_size > 1");
    if (!ctx->tables_set) return fail(ctx, B200VIS_ERR_NOT_READY, "writeback_tables: call b200vis_set_tables first");
    const bool set_visible = which & B200VIS_WB_SET_VISIBLE;
    if (set_visible && (which & B200VIS_WB_VIEW_VISIBILITY))
        return fail(ctx, B200VIS_ERR_INVALID_ARG, "writeback_tables: WB_SET_VISIBLE and WB_VIEW_VISIBILITY exclude each other");
    { const int32_t frc = flush_table_updates(ctx); if (frc) return frc; }
    // on the main stream, right behind the tile pass, like the column write-back
    const TableBufs tb{ctx->d_tabs, ctx->d_tab_chunks, ctx->n_tab_chunks, ctx->d_tab_map, ctx->d_tvv_shadow};
    if (!set_visible || (which & B200VIS_WB_GLOBAL_TRANSFORM))
        launch_writeback_tables(ctx->stream, ctx->rows, tb, which & (B200VIS_WB_GLOBAL_TRANSFORM | B200VIS_WB_VIEW_VISIBILITY), gt_tick, vv_tick);
    if (set_visible) launch_set_visible_tables(ctx->stream, ctx->rows, tb, vv_tick);
    CU(cudaGetLastError());
    return B200VIS_OK;
}

extern "C" int32_t b200vis_read_tables(b200vis_ctx *ctx, uint32_t which, uint32_t last_run, uint32_t this_run) {
    CHECK_CTX();
    if (ctx->cfg.world_size > 1) return fail(ctx, B200VIS_ERR_UNSUPPORTED, "read_tables: world_size > 1");
    if (!ctx->tables_set || ctx->h_tabs.empty()) return fail(ctx, B200VIS_ERR_NOT_READY, "read_tables: no tables are registered");
    { const int32_t frc = flush_table_updates(ctx); if (frc) return frc; }
    const TableBufs tb{ctx->d_tabs, ctx->d_tab_chunks, ctx->n_tab_chunks, ctx->d_tab_map, ctx->d_tvv_shadow};
    launch_read_tables(ctx->stream, ctx->rows, tb, which & (B200VIS_RD_TRANSFORM | B200VIS_RD_GLOBAL_TRANSFORM), last_run, this_run);
    CU(cudaGetLastError());
    if ((which & B200VIS_RD_CULL_INPUTS) && ctx->cull_attached) {
        // a read while range entries are held but not attached consumes fresh marks without writing range parameters:
        // the next attach must then read every ranged table in full, as after a detach
        if (!ctx->range_attached) ctx->h_tab_range.clear();
        const b200vis_visibility_range_layout &rl = ctx->range_layout;
        const RangeRead rr{ctx->range_attached ? ctx->d_tab_range : nullptr, rl.stride, rl.start, rl.end, rl.use_aabb,
                           ctx->d_range_se, ctx->d_range_ua};
        launch_read_table_cull(ctx->stream, ctx->rows, tb, ctx->d_tab_cull, ctx->d_tab_fresh, last_run, this_run,
                               ctx->caster_attached ? ctx->d_tab_caster : nullptr, ctx->d_caster, rr);
        CU(cudaGetLastError());
        ctx->bounds_set = true;
        // F_SPHERE_FROM_GT and HAS_AABB change on full reads only, and the host queued every one of them: the light rows
        // are verified again only then, so a steady-state read adds no synchronisation
        if (ctx->cull_fresh_pending) { ctx->lights_tag_dirty = true; ctx->cull_fresh_pending = false; }
    }
    if (which & B200VIS_RD_GLOBAL_TRANSFORM) {
        // whether a slot was newer is known only on the device: the next propagate takes the marked instantiation
        bool gt_inputs = false;
        for (const b200vis_table &t : ctx->h_tabs) gt_inputs |= t.global_transforms && t.gt_changed_ticks;
        if (gt_inputs) { ctx->gt_ext_pending = true; ctx->gt_aos_valid = false; }
    }
    return B200VIS_OK;
}

extern "C" int32_t b200vis_download_frame(b200vis_ctx *ctx, b200vis_frame_stats *stats, uint32_t *visible_rows,
                                          uint32_t visible_capacity, uint32_t *cluster_offsets,
                                          uint32_t *cluster_indices, uint32_t cluster_capacity) {
    CHECK_CTX_JOIN();
    if (!stats) return fail(ctx, B200VIS_ERR_INVALID_ARG, "download_frame: null stats");
    cudaStream_t st = ctx->stream;
    const FrameConsts &fc = active_consts(ctx);
    const uint32_t V = std::min<uint32_t>(fc.n_views, ctx->cfg.max_views);
    // sync 1: the stats block and the cluster offsets (both small, fixed size) tell how much else to copy
    CU(cudaMemcpyAsync(ctx->h_stats, ctx->d_stats, sizeof(DevStats), cudaMemcpyDeviceToHost, st));
    if (cluster_offsets)
        for (uint32_t v = 0; v < V; ++v) {
            const uint32_t nc = fc.cviews[v].enabled ? fc.cviews[v].n_clusters : 0;
            CU(cudaMemcpyAsync(cluster_offsets + (size_t)v * (kMaxClusters + 1), ctx->cl.offsets + (size_t)v * (kMaxClusters + 1),
                               (size_t)(nc + 1) * 4, cudaMemcpyDeviceToHost, st));
        }
    CU(cudaStreamSynchronize(st));
    int32_t rc = b200vis_download_frame_stats(ctx, stats);   // formats h_stats (re-copies 200 bytes)
    if (rc) return rc;
    // sync 2: exact-size list copies
    for (uint32_t v = 0; v < V; ++v) {
        if (visible_rows) {
            const uint32_t c = ctx->h_stats->visible_count[v];   // every view (b200vis_frame_stats holds the first eight)
            if (c > visible_capacity) return fail(ctx, B200VIS_ERR_CAPACITY, "download_frame: view %u has %u visible rows > capacity %u", v, c, visible_capacity);
            CU(cudaMemcpyAsync(visible_rows + (size_t)v * visible_capacity, ctx->vis.lists + (size_t)v * ctx->vis.list_stride, (size_t)c * 4, cudaMemcpyDeviceToHost, st));
        }
        if (cluster_indices && cluster_offsets && fc.cviews[v].enabled) {
            const uint32_t total = cluster_offsets[(size_t)v * (kMaxClusters + 1) + fc.cviews[v].n_clusters];
            if (total > cluster_capacity || total > ctx->cl.index_cap)
                return fail(ctx, B200VIS_ERR_CAPACITY, "download_frame: view %u has %u cluster indices > capacity", v, total);
            CU(cudaMemcpyAsync(cluster_indices + (size_t)v * cluster_capacity, ctx->cl.indices + (size_t)v * ctx->cl.index_cap, (size_t)total * 4, cudaMemcpyDeviceToHost, st));
        }
    }
    CU(cudaStreamSynchronize(st));
    return B200VIS_OK;
}

extern "C" int32_t b200vis_step(b200vis_ctx *ctx, uint32_t n_changed, const uint32_t *rows, const float *trs,
                                uint32_t n_cameras, const b200vis_camera *cameras, const b200vis_cluster_config *cfg, uint32_t flags) {
    CHECK_CTX();
    if (n_cameras > ctx->cfg.max_views || (n_cameras && !cameras)) return fail(ctx, B200VIS_ERR_INVALID_ARG, "step: bad camera array");
    int32_t rc;
    using clk = std::chrono::steady_clock;
    auto t0 = clk::now();
    auto lap = [&](int i) { auto t1 = clk::now(); ctx->step_t[i] += std::chrono::duration<double>(t1 - t0).count(); t0 = t1; };
    if (n_changed && (rc = b200vis_upload_transforms_scattered(ctx, n_changed, rows, trs))) return rc;
    lap(0);
    if ((rc = b200vis_set_view_count(ctx, n_cameras))) return rc;
    const bool clusters = cfg != nullptr && ctx->lights.n > 0;
    // frusta first, so the tile pass starts at once; the per-view cluster prologue (plane tables, z thresholds: tens of
    // microseconds of host maths) is computed while that kernel runs, then the cluster stage is enqueued behind it
    for (uint32_t v = 0; v < n_cameras; ++v)
        if ((rc = b200vis_update_camera(ctx, v, &cameras[v], nullptr, nullptr, nullptr))) return rc;
    lap(1);
    ctx->step_defers_stats = clusters;
    rc = b200vis_run(ctx, B200VIS_STAGE_PROPAGATE | B200VIS_STAGE_CULL);
    ctx->step_defers_stats = false;
    if (rc) return rc;
    if ((flags & B200VIS_STEP_WRITEBACK) && (rc = b200vis_writeback_columns(ctx))) return rc;
    lap(2);
    if (clusters) {
        for (uint32_t v = 0; v < n_cameras; ++v)
            if ((rc = b200vis_update_camera(ctx, v, &cameras[v], cfg, &ctx->auto_fb[v], nullptr))) return rc;
        lap(3);
        if ((rc = b200vis_run(ctx, B200VIS_STAGE_CLUSTER))) return rc;
        lap(4);
    }
    ctx->step_n++;
    if (!(flags & B200VIS_STEP_WAIT)) return B200VIS_OK;
    if ((rc = join_all(ctx))) return rc;
    const b200vis_frame_stats *st = nullptr;
    b200vis_frame_stats local;
    if (ctx->have_sink) { CU(cudaStreamSynchronize(ctx->stream)); st = ctx->sink.stats; }
    else { if ((rc = b200vis_download_frame_stats(ctx, &local))) return rc; st = &local; }
    lap(5);
    ctx->last_gt_changed = st->gt_changed_count;
    // views past the eighth: the view-stats sink when the result sink published this frame, else the device stats block
    // (b200vis_download_frame_stats above left a copy of it in h_stats)
    const uint32_t *wide = nullptr;
    if (clusters && n_cameras > (uint32_t)kMaxViews && ctx->have_sink) {
        if (ctx->view_stats_sink) wide = ctx->view_stats_sink;
        else {
            CU(cudaMemcpyAsync(ctx->h_stats, ctx->d_stats, sizeof(DevStats), cudaMemcpyDeviceToHost, ctx->stream));
            CU(cudaStreamSynchronize(ctx->stream));
        }
    }
    if (clusters)
        for (uint32_t v = 0; v < n_cameras; ++v) {   // Clusters::last_frame_* (assign.rs:810-811)
            b200vis_cluster_feedback &fb = ctx->auto_fb[v];
            if (!ctx->consts.cviews[v].enabled) continue;
            float far_z = 0.0f; uint32_t idx = 0;
            if (v < (uint32_t)kMaxViews) { far_z = st->cluster_farthest_z[v]; idx = st->cluster_index_count[v]; }
            else if (wide) { memcpy(&far_z, &wide[(size_t)v * 4 + 2], 4); idx = wide[(size_t)v * 4 + 1]; }
            else { memcpy(&far_z, &ctx->h_stats->cl_farthest_bits[v], 4); idx = ctx->h_stats->cl_index_count[v]; }
            fb.has_farthest_z = 1; fb.farthest_z = far_z;
            fb.has_index_count = 1; fb.index_count = idx;
        }
    return B200VIS_OK;
}
