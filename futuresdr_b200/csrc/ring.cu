// ring.cu -- device-resident stream-buffer ring (the CUDA counterpart of the reference's
// accelerator buffers: src/runtime/buffer/vulkan/{h2d,d2h}.rs, circuit.rs, and the history
// prefix of slab.rs:370-398).
//
// n_slots buffers live in HBM for the lifetime of the ring; what moves between blocks is
// OWNERSHIP of a slot, through two FIFOs -- `empty` (the circuit's inbound queue,
// h2d.rs:161-197) and `full` (outbound, h2d.rs:199-232 / d2h.rs:66-74).  A slot is
//   [ pad | halo_items | chunk_items ]            (data start 256-byte aligned)
// so a FIR block sees its (ntaps-1) samples of history contiguously in front of the new chunk
// without the samples ever leaving the device; b2s_ring_carry_halo copies the unconsumed tail
// of the previous slot there (what slab.rs does on the CPU).  With host staging each slot also
// owns a pinned buffer for the H2D / D2H edges (VectorSource<H2DWriter> / VectorSink<D2HReader>
// in tests/vulkan.rs:56-66).  Each slot carries a CUDA event so edges and other streams can
// wait for the work that produced it (the Vulkan fence, blocks/vulkan.rs:157-162).
#include <deque>

#include "common.cuh"

enum SlotState { SLOT_EMPTY = 0, SLOT_HELD_EMPTY = 1, SLOT_FULL = 2, SLOT_HELD_FULL = 3 };

struct b2s_slot {
    b2s_ring *ring = nullptr;
    int index = 0;
    char *d_data = nullptr;        // first data item (halo is below)
    char *h_stage = nullptr;
    cudaEvent_t ev = nullptr;
    size_t valid = 0, halo_valid = 0;
    SlotState state = SLOT_EMPTY;
};

struct b2s_ring {
    b2s_ctx *ctx = nullptr;
    size_t item_bytes = 0, chunk_items = 0, halo_items = 0;
    std::vector<b2s_slot> slots;
    std::deque<int> empty, full;
    mutable std::mutex mu;
    Buf<char> d_mem;
    Buf<char, Mem::Pinned> h_mem;
    size_t slot_bytes = 0, halo_bytes = 0, total_bytes = 0, flags_off = 0;

    ~b2s_ring() {
        for (auto &s : slots) if (s.ev) cudaEventDestroy(s.ev);
    }
};

extern "C" {

int32_t b2s_ring_create(b2s_ctx *ctx, size_t item_bytes, size_t chunk_items, size_t halo_items,
                        int32_t n_slots, int32_t with_host_staging, b2s_ring **out) {
    if (!ctx || !out) return b2s_fail(ctx, B2S_EINVAL, "b2s_ring_create: NULL argument");
    *out = nullptr;
    if (item_bytes == 0 || chunk_items == 0 || n_slots < 1 || n_slots > 1024)
        return b2s_fail(ctx, B2S_EINVAL, "b2s_ring_create: bad geometry");
    DeviceGuard g(ctx->device);
    PlanPtr<b2s_ring> r(new b2s_ring());
    r->ctx = ctx; r->item_bytes = item_bytes; r->chunk_items = chunk_items; r->halo_items = halo_items;
    const size_t halo_bytes = round_up(halo_items * item_bytes, 256);
    const size_t data_bytes = round_up(chunk_items * item_bytes, 256);
    const size_t slot_bytes = halo_bytes + data_bytes;
    // ONE allocation (so one CUDA-IPC handle exports the whole ring to a peer process): slots, then 256 bytes of
    // system-scope flags {ready, consumed} for the cross-GPU halo handshake (peer.cu)
    r->slot_bytes = slot_bytes; r->halo_bytes = halo_bytes; r->flags_off = slot_bytes * n_slots;
    r->total_bytes = r->flags_off + 256;
    B2S_TRY(r->d_mem.alloc(ctx, r->total_bytes, "ring device memory"));
    cudaMemsetAsync(r->d_mem.get() + r->flags_off, 0, 256, ctx->stream);
    if (with_host_staging) B2S_TRY(r->h_mem.alloc(ctx, data_bytes * n_slots, "ring pinned staging"));
    r->slots.resize(n_slots);
    for (int i = 0; i < n_slots; i++) {
        b2s_slot &s = r->slots[i];
        s.ring = r.get(); s.index = i;
        s.d_data = r->d_mem.get() + (size_t)i * slot_bytes + halo_bytes;
        s.h_stage = r->h_mem ? r->h_mem.get() + (size_t)i * data_bytes : nullptr;
        B2S_CUDA(ctx, cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming));
        r->empty.push_back(i);
    }
    *out = r.release();
    return B2S_OK;
}

void b2s_ring_destroy(b2s_ring *r) { PlanDeleter<b2s_ring>()(r); }

int32_t b2s_ring_acquire_empty(b2s_ring *r, b2s_slot **slot) {
    if (!r || !slot) return b2s_fail(r ? r->ctx : nullptr, B2S_EINVAL, "b2s_ring_acquire_empty: NULL argument");
    std::lock_guard<std::mutex> lk(r->mu);
    if (r->empty.empty()) { *slot = nullptr; return B2S_EAGAIN; }
    b2s_slot &s = r->slots[r->empty.front()];
    r->empty.pop_front();
    s.state = SLOT_HELD_EMPTY; s.valid = 0; s.halo_valid = 0;
    *slot = &s;
    return B2S_OK;
}

int32_t b2s_ring_submit_full(b2s_ring *r, b2s_slot *slot, size_t valid_items, int32_t from_host) {
    if (!r || !slot || slot->ring != r) return b2s_fail(r ? r->ctx : nullptr, B2S_EINVAL, "b2s_ring_submit_full: bad slot");
    if (slot->state != SLOT_HELD_EMPTY) return b2s_fail(r->ctx, B2S_ESTATE, "b2s_ring_submit_full: slot %d is not held empty", slot->index);
    if (valid_items > r->chunk_items) return b2s_fail(r->ctx, B2S_EINVAL, "b2s_ring_submit_full: %zu items > chunk %zu", valid_items, r->chunk_items);
    DeviceGuard g(r->ctx->device);
    if (from_host) {
        if (!slot->h_stage) return b2s_fail(r->ctx, B2S_ESTATE, "b2s_ring_submit_full: ring has no host staging");
        B2S_CUDA(r->ctx, cudaMemcpyAsync(slot->d_data, slot->h_stage, valid_items * r->item_bytes,
                                         cudaMemcpyHostToDevice, r->ctx->stream));
    }
    B2S_CUDA(r->ctx, cudaEventRecord(slot->ev, r->ctx->stream));
    std::lock_guard<std::mutex> lk(r->mu);
    slot->valid = valid_items;
    slot->state = SLOT_FULL;
    r->full.push_back(slot->index);
    return B2S_OK;
}

int32_t b2s_ring_acquire_full(b2s_ring *r, b2s_slot **slot, size_t *valid_items) {
    if (!r || !slot) return b2s_fail(r ? r->ctx : nullptr, B2S_EINVAL, "b2s_ring_acquire_full: NULL argument");
    b2s_slot *s = nullptr;
    {
        std::lock_guard<std::mutex> lk(r->mu);
        if (r->full.empty()) { *slot = nullptr; if (valid_items) *valid_items = 0; return B2S_EAGAIN; }
        s = &r->slots[r->full.front()];
        r->full.pop_front();
        s->state = SLOT_HELD_FULL;
    }
    DeviceGuard g(r->ctx->device);
    B2S_CUDA(r->ctx, cudaStreamWaitEvent(r->ctx->stream, s->ev, 0));   // producer may be another stream
    *slot = s;
    if (valid_items) *valid_items = s->valid;
    return B2S_OK;
}

int32_t b2s_ring_release(b2s_ring *r, b2s_slot *slot) {
    if (!r || !slot || slot->ring != r) return b2s_fail(r ? r->ctx : nullptr, B2S_EINVAL, "b2s_ring_release: bad slot");
    if (slot->state != SLOT_HELD_FULL && slot->state != SLOT_HELD_EMPTY)
        return b2s_fail(r->ctx, B2S_ESTATE, "b2s_ring_release: slot %d is not held", slot->index);
    DeviceGuard g(r->ctx->device);
    // whoever refills the slot must wait for the work that last read it
    B2S_CUDA(r->ctx, cudaEventRecord(slot->ev, r->ctx->stream));
    std::lock_guard<std::mutex> lk(r->mu);
    slot->state = SLOT_EMPTY; slot->valid = 0; slot->halo_valid = 0;
    r->empty.push_back(slot->index);
    return B2S_OK;
}

int32_t b2s_ring_carry_halo(b2s_ring *r, const b2s_slot *from, size_t from_valid, size_t tail_items, b2s_slot *to) {
    if (!r || !from || !to || from->ring != r || to->ring != r) return b2s_fail(r ? r->ctx : nullptr, B2S_EINVAL, "b2s_ring_carry_halo: bad slot");
    if (tail_items > r->halo_items) return b2s_fail(r->ctx, B2S_EINVAL, "b2s_ring_carry_halo: tail %zu > halo %zu", tail_items, r->halo_items);
    if (tail_items > from_valid + from->halo_valid) return b2s_fail(r->ctx, B2S_EINVAL, "b2s_ring_carry_halo: tail longer than the source slot");
    DeviceGuard g(r->ctx->device);
    if (tail_items) {
        // the tail may itself reach back into `from`'s own halo (chunks shorter than the history)
        const char *src = from->d_data + ((long long)from_valid - (long long)tail_items) * (long long)r->item_bytes;
        B2S_CUDA(r->ctx, cudaMemcpyAsync(to->d_data - tail_items * r->item_bytes, src, tail_items * r->item_bytes,
                                         cudaMemcpyDeviceToDevice, r->ctx->stream));
    }
    to->halo_valid = tail_items;
    return B2S_OK;
}

void *b2s_slot_device_ptr(const b2s_slot *s) { return s ? s->d_data : nullptr; }
void *b2s_slot_host_ptr(const b2s_slot *s) { return s ? s->h_stage : nullptr; }
size_t b2s_slot_halo_valid(const b2s_slot *s) { return s ? s->halo_valid : 0; }

int32_t b2s_slot_fetch_to_host(b2s_slot *s, size_t items) {
    if (!s) return b2s_fail(nullptr, B2S_EINVAL, "slot is NULL");
    b2s_ring *r = s->ring;
    if (!s->h_stage) return b2s_fail(r->ctx, B2S_ESTATE, "b2s_slot_fetch_to_host: ring has no host staging");
    if (items > r->chunk_items) return b2s_fail(r->ctx, B2S_EINVAL, "b2s_slot_fetch_to_host: too many items");
    DeviceGuard g(r->ctx->device);
    B2S_CUDA(r->ctx, cudaMemcpyAsync(s->h_stage, s->d_data, items * r->item_bytes, cudaMemcpyDeviceToHost, r->ctx->stream));
    B2S_CUDA(r->ctx, cudaEventRecord(s->ev, r->ctx->stream));
    return B2S_OK;
}

int32_t b2s_slot_wait(b2s_slot *s) {
    if (!s) return b2s_fail(nullptr, B2S_EINVAL, "slot is NULL");
    DeviceGuard g(s->ring->ctx->device);
    B2S_CUDA(s->ring->ctx, cudaEventSynchronize(s->ev));
    return B2S_OK;
}

void *b2s_ring_base(const b2s_ring *r) { return r ? r->d_mem.get() : nullptr; }
size_t b2s_ring_bytes(const b2s_ring *r) { return r ? r->total_bytes : 0; }
size_t b2s_ring_slot_offset(const b2s_ring *r, int32_t slot_index) {
    if (!r || slot_index < 0 || (size_t)slot_index >= r->slots.size()) return 0;
    return (size_t)slot_index * r->slot_bytes + r->halo_bytes;
}
size_t b2s_ring_flags_offset(const b2s_ring *r) { return r ? r->flags_off : 0; }
int32_t b2s_slot_index(const b2s_slot *s) { return s ? s->index : -1; }

size_t b2s_ring_free_slots(const b2s_ring *r) {
    if (!r) return 0;
    std::lock_guard<std::mutex> lk(r->mu);
    return r->empty.size();
}
size_t b2s_ring_full_slots(const b2s_ring *r) {
    if (!r) return 0;
    std::lock_guard<std::mutex> lk(r->mu);
    return r->full.size();
}

}  // extern "C"
