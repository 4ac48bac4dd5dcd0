// r3_batching.cpp — host side of GpuCuller::add_culling_to_graph: batch_objects
// (rend3-routine/src/culling/batching.rs:120-250) over the visible list produced on the GPU.
//
// The reference runs this single-threaded on the CPU for every camera; it stays host code here
// (SURVEY 8f ranks a device-side sort/batch build as the next row).  Differences from the reference:
// the frustum filter (batching.rs:144-148) already ran on the GPU, and ties in the unstable sort are
// resolved by object handle so that the result is deterministic.
#include <algorithm>
#include <cstring>

#include "r3_common.cuh"

namespace {
struct SortItem {
    uint64_t material_key;
    uint32_t reason;     // SortingReason: Optimization = 0 < Requirement = 1 (rend3-types/src/lib.rs:952-957)
    float distance;      // OrderedFloat<f32>; negated for BackToFront (batching.rs:158-160)
    uint32_t handle;
};
// ShaderJobSortingKey::cmp (batching.rs:53-79) with bind_group_index == DUMMY everywhere (GpuDriven profile)
inline bool sort_less(const SortItem& a, const SortItem& b) {
    if (a.material_key != b.material_key) return a.material_key < b.material_key;
    if (a.reason != b.reason) return a.reason < b.reason;
    // OrderedFloat: NaN is greater than every number and equal to itself, -0.0 == +0.0 — a strict weak order for std::sort
    const bool an = a.distance != a.distance, bn = b.distance != b.distance;
    if (an != bn) return bn;
    if (!an) {
        if (a.distance < b.distance) return true;
        if (a.distance > b.distance) return false;
    }
    return a.handle < b.handle;
}
inline uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }

// index_count of every visible object, so the host never needs a copy of the object records
__global__ void gather_index_count_kernel(const r3_object* __restrict__ objects, const uint32_t* __restrict__ visible, uint32_t n,
                                          uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = objects[visible[i]].index_count;
}
}  // namespace

int r3_host_batch_objects(r3_ctx* c, r3_camera* cam, const float vp_loc[3], uint32_t max_dispatch_count) {
    if (!cam->header_set) return r3_fail(c, R3_E_STATE, "batch_objects before object_uniform_upload");
    const uint32_t cap = cam->header.object_count;
    if (c->sort_key.size() < cap) return r3_fail(c, R3_E_STATE, "batch_objects needs r3_set_object_sort_info");
    // visible list: the only device->host transfer of the frame (4 B per visible object), and with it the locations of the objects
    // r3_pose_objects posed since the host mirror last took them (12 B per posed object) and, after r3_set_object_transforms / _device,
    // every location (12 B per slot: the host does not know which slots a device list named), so that no extra drain is needed
    uint32_t nv = 0;
    // and, after r3_switch_object_variants_device, the listed slots' current variants (4 B per slot), from which the key mirrors follow
    bool mirrors = false;
    R3_TRY(r3_stage_sort_mirrors(c, &mirrors));
    if (cam->d_visible_count || mirrors) {
        if (cam->d_visible_count) R3_CUDA(c, cudaMemcpyAsync(&nv, cam->d_visible_count, 4, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
    }
    if (mirrors) r3_apply_sort_mirrors(c);
    cam->visible_count_host = (int)nv;
    std::vector<uint32_t> visible(nv), index_count(nv);
    if (nv) {
        R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, (uint64_t)nv * 4, 1, false, false));
        gather_index_count_kernel<<<(nv + 255) / 256, 256, 0, c->stream>>>(c->d_objects, cam->d_visible, nv, (uint32_t*)c->d_scratch);
        R3_CHECK_LAUNCH(c, "gather_index_count_kernel");
        R3_CUDA(c, cudaMemcpyAsync(visible.data(), cam->d_visible, (size_t)nv * 4, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, cudaMemcpyAsync(index_count.data(), c->d_scratch, (size_t)nv * 4, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
    }
    std::vector<SortItem> items(nv);
    for (uint32_t i = 0; i < nv; ++i) {
        const uint32_t h = visible[i];
        const float* l = &c->sort_loc[3 * (size_t)h];
        const float dx = vp_loc[0] - l[0], dy = vp_loc[1] - l[1], dz = vp_loc[2] - l[2];
        float d2 = (dx * dx + dy * dy) + dz * dz;                 // Vec3A::distance_squared (batching.rs:156-157)
        if (c->sort_flags[h] & 4) d2 = -d2;
        items[i] = SortItem{c->sort_key[h], (c->sort_flags[h] & 2) ? 0u : 1u, d2, h};
    }
    std::vector<uint32_t> order(nv);   // index_count follows its object through the sort
    for (uint32_t i = 0; i < nv; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return sort_less(items[a], items[b]); });

    const int w = (cam->cache_idx == 0) ? 1 : 0;   // never overwrite the DrawCallSet cached for the predicted pass
    cam->cur = w;
    r3_jobs& jobs = cam->jobs[w];
    jobs.batches.clear(); jobs.regions.clear(); jobs.total_invocations = 0; jobs.valid = false; jobs.device_built = false;

    std::vector<uint32_t> cur_map(cap, R3_NO_PREVIOUS);          // get_and_reset_camera / set_camera (batching.rs:111-117)
    const std::vector<uint32_t>& prev_map = cam->prev_invocation;
    if (nv) {
        uint32_t cur_region_idx = 0, cur_region_obj = 0, cur_base_inv = 0, cur_region_inv = 0, cur_inv = 0, cur_obj = 0;
        uint64_t cur_key = items[order[0]].material_key;
        r3_batch_data cur;
        std::memset(&cur, 0, sizeof cur);
        auto push_region = [&](uint64_t key) { jobs.regions.push_back(r3_region{(uint32_t)jobs.batches.size(), 0u, key}); };
        auto push_batch = [&]() {
            cur.total_objects = cur_obj; cur.total_invocations = cur_inv; cur.batch_base_invocation = cur_base_inv;
            jobs.batches.push_back(cur);
        };
        for (uint32_t oi = 0; oi < nv; ++oi) {
            const uint32_t i = order[oi];
            const uint32_t h = items[i].handle;
            const uint32_t invocation_count = index_count[i] / 3;
            const bool key_difference = items[i].material_key != cur_key;
            const bool object_limit = cur_obj == R3_BATCH_SIZE;
            const bool dispatch_limit = ((uint64_t)cur_inv + invocation_count) >= (uint64_t)max_dispatch_count * R3_WORKGROUP_SIZE;
            if (key_difference || object_limit || dispatch_limit) {
                push_region(cur_key);
                cur_region_idx += 1; cur_key = items[i].material_key; cur_region_obj = 0; cur_region_inv = cur_inv;
            }
            if (object_limit || dispatch_limit) {
                push_batch();
                cur_base_inv += cur_inv; cur_inv = 0; cur_region_inv = 0; cur_obj = 0;
            }
            r3_object_culling_info& r = cur.object_culling_information[cur_obj];
            r.invocation_start = cur_inv;
            r.invocation_end = cur_inv + invocation_count;
            r.region_id = cur_region_idx;
            r.object_id = h;
            r.base_region_invocation = cur_region_inv;
            r.local_region_id = cur_region_obj;
            r.previous_global_invocation = h < prev_map.size() ? prev_map[h] : R3_NO_PREVIOUS;
            r.atomic_capable = (c->sort_flags[h] & 2) ? 1u : 0u;
            cur_map[h] = cur_inv + cur_base_inv;
            cur_obj += 1; cur_region_obj += 1;
            cur_inv += round_up(invocation_count, R3_WORKGROUP_SIZE);
        }
        push_region(cur_key);
        push_batch();
        uint64_t tot = 0;
        for (const auto& b : jobs.batches) tot += b.total_invocations;
        jobs.total_invocations = (uint32_t)tot;
    }
    cam->prev_invocation.swap(cur_map);
    return R3_OK;
}

// copies jobs[cur] to the device and derives each region's first global invocation
int r3_upload_jobs(r3_ctx* c, r3_camera* cam) {
    r3_jobs& j = cam->jobs[cam->cur];
    const uint32_t nb = (uint32_t)j.batches.size(), nr = (uint32_t)j.regions.size();
    R3_TRY(r3_reserve_t(c, &j.d_batches, &j.batches_cap, nb));
    uint32_t rcap = j.regions_cap;
    R3_TRY(r3_reserve_t(c, &j.d_regions, &j.regions_cap, nr));
    if (!j.d_region_first_inv || rcap != j.regions_cap) {
        cudaFree(j.d_region_first_inv);
        j.d_region_first_inv = nullptr;
        R3_CUDA(c, cudaMalloc((void**)&j.d_region_first_inv, ((size_t)j.regions_cap + 2) * 4));
    }
    std::vector<uint32_t> first(nr + 1, 0u);
    for (const auto& b : j.batches)
        for (uint32_t o = 0; o < b.total_objects && o < R3_BATCH_SIZE; ++o) {
            const r3_object_culling_info& info = b.object_culling_information[o];
            if (info.local_region_id == 0 && info.region_id < nr) first[info.region_id] = b.batch_base_invocation + info.invocation_start;
        }
    first[nr] = j.total_invocations;
    R3_CUDA(c, cudaMemcpyAsync(j.d_batches, j.batches.data(), (size_t)nb * sizeof(r3_batch_data), cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(j.d_regions, j.regions.data(), (size_t)nr * sizeof(r3_region), cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(j.d_region_first_inv, first.data(), ((size_t)nr + 1) * 4, cudaMemcpyHostToDevice, c->stream));
    if (!j.d_header) R3_CUDA(c, cudaMalloc((void**)&j.d_header, 32));
    const uint32_t hdr[8] = {(uint32_t)(cam->visible_count_host < 0 ? 0 : cam->visible_count_host), nb, nr, j.total_invocations, 0, 0, 0, 0};
    R3_CUDA(c, cudaMemcpyAsync(j.d_header, hdr, 32, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));   // `first` and the vectors are pageable host memory
    j.n_batches = nb; j.n_regions = nr; j.valid = true;
    return R3_OK;
}
