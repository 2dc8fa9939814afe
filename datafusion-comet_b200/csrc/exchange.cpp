// exchange.cpp -- the one real exchange step of the hot path: hash-repartitioned aggregate state between the GPUs of one box.
//
// The reference writes the rows of every output partition as IPC blocks to local files and the reduce side fetches them
// (native/shuffle/src/partitioners/multi_partition.rs:265-330 + Spark's block transfer).  With one process per GPU on one box the
// same rows travel over NVLink / NVSwitch instead: the map side (PartitionNode, partition.cpp) leaves every column reordered by
// partition id on the device, and cb200_exchange moves segment p of every column to rank p --
//   counts : one ncclAllGather of the N x N row-count matrix (the "map status" Spark's driver would collect)
//   payload: ONE ncclGroup of N sends + N receives per column buffer, straight out of the map plan's device buffers into the buffers
//            the Final plan will read (no staging copy, no host hop)
// NCCL is loaded at run time (dlopen): inside a torchrun worker that resolves to the libnccl torch already mapped, elsewhere to the
// system library.  Nothing else in the library depends on it.
#include "../../include/comet_b200.h"

#include "abi_internal.h"
#include "exec.h"

#include <dlfcn.h>
#include <nccl.h>

#include <cstring>
#include <mutex>

using namespace cb200;

namespace {

struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
    void* handle = nullptr;
    std::string where;
};

NcclApi& nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            api.handle = dlopen(n, RTLD_NOW | RTLD_NOLOAD); // the copy the host process already uses (torch bundles one)
            if (api.handle) { api.where = std::string(n) + " (already loaded)"; break; }
        }
        if (!api.handle)
            for (const char* n : names) {
                api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
                if (api.handle) { api.where = n; break; }
            }
        if (!api.handle) return;
        auto sym = [&](const char* s) { return dlsym(api.handle, s); };
        api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
        api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
        api.Send = (decltype(api.Send))sym("ncclSend");
        api.Recv = (decltype(api.Recv))sym("ncclRecv");
        api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
        api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
        api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
        api.GetVersion = (decltype(api.GetVersion))sym("ncclGetVersion");
    });
    if (!api.handle || !api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.Send || !api.Recv || !api.GroupStart || !api.GroupEnd)
        throw ExecError(CB200_ERR_CUDA, "", "NCCL is not available (libnccl.so.2 could not be loaded): the multi-GPU exchange needs it");
    return api;
}

void nccl_check(ncclResult_t r, const char* what) {
    if (r != ncclSuccess) {
        NcclApi& a = nccl();
        throw ExecError(CB200_ERR_CUDA, "", std::string("NCCL error in ") + what + ": " + (a.GetErrorString ? a.GetErrorString(r) : "?"));
    }
}

} // namespace

struct cb200_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ready = nullptr;
    int64_t* d_counts = nullptr;   // [world] send counts + [world * world] gathered
    int64_t* h_counts = nullptr;   // pinned mirror
    uint8_t *d_small = nullptr, *h_small = nullptr; // small-payload all-gather (aggregate states of dense / ungrouped plans)
    size_t small_cap = 0;
};

extern "C" {

int cb200_comm_unique_id(uint8_t* id_out, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        static_assert(sizeof(ncclUniqueId) <= CB200_UNIQUE_ID_BYTES, "unique id size");
        ncclUniqueId id;
        nccl_check(nccl().GetUniqueId(&id), "ncclGetUniqueId");
        memset(id_out, 0, CB200_UNIQUE_ID_BYTES);
        memcpy(id_out, &id, sizeof(id));
        return 0;
    }, -1);
}

cb200_comm* cb200_comm_create(const uint8_t* id_bytes, int32_t rank, int32_t world, int32_t device, cb200_error* err) {
    return cb200_guarded(err, [&]() -> cb200_comm* {
        if (world < 1 || rank < 0 || rank >= world) throw PlanError("cb200_comm_create: bad rank / world");
        auto c = std::unique_ptr<cb200_comm>(new cb200_comm());
        c->rank = rank;
        c->world = world;
        c->device = device;
        cuda_check(cudaSetDevice(device), "cudaSetDevice");
        cuda_check(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking), "comm stream");
        cuda_check(cudaEventCreate(&c->ev0), "event");
        cuda_check(cudaEventCreate(&c->ev1), "event");
        cuda_check(cudaEventCreateWithFlags(&c->ready, cudaEventDisableTiming), "event");
        const size_t n = (size_t)world + (size_t)world * world;
        cuda_check(cudaMalloc((void**)&c->d_counts, n * 8), "cudaMalloc counts");
        cuda_check(cudaMallocHost((void**)&c->h_counts, n * 8), "cudaMallocHost counts");
        if (world > 1) {
            ncclUniqueId id;
            memcpy(&id, id_bytes, sizeof(id));
            nccl_check(nccl().CommInitRank(&c->comm, world, id, rank), "ncclCommInitRank");
        }
        return c.release();
    }, (cb200_comm*)nullptr);
}

void cb200_comm_destroy(cb200_comm* c) {
    if (!c) return;
    try {
        cudaSetDevice(c->device);
        if (c->stream) cudaStreamSynchronize(c->stream);
        if (c->comm) nccl().CommDestroy(c->comm);
        if (c->d_counts) cudaFree(c->d_counts);
        if (c->h_counts) cudaFreeHost(c->h_counts);
        if (c->d_small) cudaFree(c->d_small);
        if (c->h_small) cudaFreeHost(c->h_small);
        if (c->ev0) cudaEventDestroy(c->ev0);
        if (c->ev1) cudaEventDestroy(c->ev1);
        if (c->ready) cudaEventDestroy(c->ready);
        if (c->stream) cudaStreamDestroy(c->stream);
    } catch (...) {
    }
    delete c;
}

int32_t cb200_comm_rank(cb200_comm* c) { return c ? c->rank : -1; }
int32_t cb200_comm_world(cb200_comm* c) { return c ? c->world : -1; }

// receive offsets of an all-to-all from the gathered count matrix: rank `me` receives counts[s * world + me] rows from rank s, in
// rank order (so the received rows of one source stay contiguous and in their map-side order)
int64_t cb200_exchange_layout(const int64_t* counts, int32_t world, int32_t me, int64_t* recv_counts, int64_t* recv_offsets) {
    int64_t total = 0;
    for (int s = 0; s < world; s++) {
        const int64_t c = counts[(size_t)s * world + me];
        if (recv_counts) recv_counts[s] = c;
        if (recv_offsets) recv_offsets[s] = total;
        total += c;
    }
    return total;
}

cb200_table* cb200_exchange(cb200_comm* c, cb200_plan* plan, int64_t* n_rows_out, cb200_exchange_stats* stats, cb200_error* err) {
    return cb200_guarded(err, [&]() -> cb200_table* {
        if (!c || !plan) throw PlanError("cb200_exchange: null handle");
        TraceSpan ts("exchange");
        const int world = c->world, me = c->rank;
        const std::vector<int64_t>& starts = cb200_plan_ctx(plan).partition_starts;
        Batch& b = cb200_plan_last(plan);
        if ((int)starts.size() != world + 1) throw PlanError("cb200_exchange: the plan's last batch has " + std::to_string(starts.empty() ? 0 : starts.size() - 1) + " partitions, the communicator " + std::to_string(world) + " ranks (run a ShuffleWriter plan with num_partitions = world size first)");
        cuda_check(cudaSetDevice(c->device), "cudaSetDevice");
        cudaStream_t st = c->stream;
        // the map plan's kernels are done (cb200_execute* synchronises), but order the streams explicitly anyway
        cuda_check(cudaEventRecord(c->ready, cb200_plan_ctx(plan).stream), "event record");
        cuda_check(cudaStreamWaitEvent(st, c->ready, 0), "stream wait");
        // ---- counts: the N x N matrix of rows rank s holds for rank p --------------------------------------------------------------
        std::vector<int64_t> recv_counts((size_t)world), recv_off((size_t)world);
        int64_t n_recv = 0;
        for (int p = 0; p < world; p++) c->h_counts[p] = starts[(size_t)p + 1] - starts[(size_t)p];
        if (world > 1) {
            cuda_check(cudaMemcpyAsync(c->d_counts, c->h_counts, (size_t)world * 8, cudaMemcpyHostToDevice, st), "counts H2D");
            nccl_check(nccl().AllGather(c->d_counts, c->d_counts + world, (size_t)world, ncclInt64, c->comm, st), "ncclAllGather(counts)");
            cuda_check(cudaMemcpyAsync(c->h_counts + world, c->d_counts + world, (size_t)world * world * 8, cudaMemcpyDeviceToHost, st), "counts D2H");
            cuda_check(cudaStreamSynchronize(st), "counts sync");
            n_recv = cb200_exchange_layout(c->h_counts + world, world, me, recv_counts.data(), recv_off.data());
        } else {
            recv_counts[0] = c->h_counts[0];
            recv_off[0] = 0;
            n_recv = recv_counts[0];
        }
        // ---- receive buffers = the Final plan's input table ------------------------------------------------------------------------------
        set_alloc_stream(st);
        auto table = std::make_shared<DeviceTable>();
        table->n_rows = n_recv;
        struct Move { const char* src; char* dst; size_t w; };
        std::vector<Move> moves;
        const size_t alloc_rows = (size_t)std::max<int64_t>(n_recv, 1);
        int64_t bytes_sent = 0, bytes_recv = 0;
        for (auto& col : b.cols) {
            if (col.on_host) throw Unsupported("exchange of host-resident columns (small dense aggregate states are gathered, not exchanged)");
            if (col.is_dict) throw Unsupported("exchange of dictionary-coded string columns (per-rank dictionaries differ)");
            if (col.offsets) throw Unsupported("exchange of plain string columns");
            Column o;
            o.type = col.type;
            o.phys = col.phys;
            o.null_count = col.validity || col.valid_bytes ? -1 : 0;
            const bool is_bool = col.type.id == TypeId::Bool;
            if (is_bool) {
                if (!col.bool_bytes) throw ExecError(15, "", "internal: boolean column of a ShuffleWriter batch without its byte form");
                o.bool_bytes = std::make_shared<DeviceBuf>(alloc_rows + 16);
                o.phys = Phys::Bitmap;
                moves.push_back({(const char*)col.bool_bytes->ptr, (char*)o.bool_bytes->ptr, 1});
                table->needs_packing = true;
            } else {
                const size_t w = (size_t)phys_bytes(col.phys);
                if (w == 0 || !col.data) throw ExecError(15, "", "internal: column without a fixed-width device form in an exchange");
                o.data = std::make_shared<DeviceBuf>(alloc_rows * w + 16);
                moves.push_back({(const char*)col.data->ptr, (char*)o.data->ptr, w});
            }
            if (col.validity) {
                if (!col.valid_bytes) throw ExecError(15, "", "internal: nullable column of a ShuffleWriter batch without byte-per-row validity");
                o.valid_bytes = std::make_shared<DeviceBuf>(alloc_rows + 16);
                moves.push_back({(const char*)col.valid_bytes->ptr, (char*)o.valid_bytes->ptr, 1});
                table->needs_packing = true;
            }
            table->cols.push_back(o);
        }
        // ---- payload: per buffer, segment p -> rank p --------------------------------------------------------------------------------------
        cuda_check(cudaEventRecord(c->ev0, st), "event record");
        if (world > 1) {
            nccl_check(nccl().GroupStart(), "ncclGroupStart");
            for (auto& m : moves)
                for (int p = 0; p < world; p++) {
                    const size_t sb = (size_t)(starts[(size_t)p + 1] - starts[(size_t)p]) * m.w, rb = (size_t)recv_counts[(size_t)p] * m.w;
                    if (sb) nccl_check(nccl().Send(m.src + (size_t)starts[(size_t)p] * m.w, sb, ncclInt8, p, c->comm, st), "ncclSend");
                    if (rb) nccl_check(nccl().Recv(m.dst + (size_t)recv_off[(size_t)p] * m.w, rb, ncclInt8, p, c->comm, st), "ncclRecv");
                    bytes_sent += (int64_t)sb;
                    bytes_recv += (int64_t)rb;
                }
            nccl_check(nccl().GroupEnd(), "ncclGroupEnd");
        } else {
            for (auto& m : moves) {
                const size_t nb = (size_t)n_recv * m.w;
                if (nb) cuda_check(cudaMemcpyAsync(m.dst, m.src, nb, cudaMemcpyDeviceToDevice, st), "local partition copy");
                bytes_sent += (int64_t)nb;
                bytes_recv += (int64_t)nb;
            }
        }
        cuda_check(cudaEventRecord(c->ev1, st), "event record");
        cuda_check(cudaStreamSynchronize(st), "exchange sync"); // the map plan may be released and the table bound right after this call
        if (n_rows_out) *n_rows_out = n_recv;
        if (stats) {
            float ms = 0;
            cudaEventElapsedTime(&ms, c->ev0, c->ev1);
            stats->rows_sent = starts[(size_t)world] - starts[0];
            stats->rows_received = n_recv;
            stats->bytes_sent = bytes_sent;
            stats->bytes_received = bytes_recv;
            stats->payload_ms = ms;
        }
        auto* t = cb200_table_wrap(table);
        return t;
    }, (cb200_table*)nullptr);
}

// All-gather of one small host payload per rank (the serialized state batch of a dense / ungrouped Partial aggregate: a few rows).
// out = world slots of `slot_bytes` each, lengths in sizes_out.  One collective, one synchronisation, no pickling.
int cb200_comm_allgather_small(cb200_comm* c, const void* payload, int64_t n_bytes, int64_t slot_bytes, void* out, int64_t* sizes_out, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        if (!c) throw PlanError("null communicator");
        if (n_bytes < 0 || slot_bytes < 16 || n_bytes + 8 > slot_bytes || (slot_bytes & 15)) throw PlanError("cb200_comm_allgather_small: payload does not fit its slot (slot_bytes must be a multiple of 16 and >= n_bytes + 8)");
        const int world = c->world, me = c->rank;
        const size_t total = (size_t)slot_bytes * world;
        cuda_check(cudaSetDevice(c->device), "cudaSetDevice");
        if (c->small_cap < total) {
            if (c->d_small) cudaFree(c->d_small);
            if (c->h_small) cudaFreeHost(c->h_small);
            c->d_small = c->h_small = nullptr;
            cuda_check(cudaMalloc((void**)&c->d_small, 2 * total), "cudaMalloc small");
            cuda_check(cudaMallocHost((void**)&c->h_small, 2 * total), "cudaMallocHost small");
            c->small_cap = total;
        }
        uint8_t* mine = c->h_small + total + (size_t)slot_bytes * me; // second half of the pinned block: staging of this rank's slot
        memcpy(mine, &n_bytes, 8);
        if (n_bytes) memcpy(mine + 8, payload, (size_t)n_bytes);
        if (world > 1) {
            uint8_t* d_mine = c->d_small + total;
            cuda_check(cudaMemcpyAsync(d_mine, mine, (size_t)slot_bytes, cudaMemcpyHostToDevice, c->stream), "small H2D");
            nccl_check(nccl().AllGather(d_mine, c->d_small, (size_t)slot_bytes, ncclInt8, c->comm, c->stream), "ncclAllGather(small)");
            cuda_check(cudaMemcpyAsync(c->h_small, c->d_small, total, cudaMemcpyDeviceToHost, c->stream), "small D2H");
            cuda_check(cudaStreamSynchronize(c->stream), "small sync");
        } else {
            memcpy(c->h_small, mine, (size_t)slot_bytes);
        }
        for (int r = 0; r < world; r++) {
            int64_t len;
            memcpy(&len, c->h_small + (size_t)slot_bytes * r, 8);
            if (len < 0 || len + 8 > slot_bytes) throw ExecError(CB200_ERR_CUDA, "", "cb200_comm_allgather_small: corrupt slot header");
            if (sizes_out) sizes_out[r] = len;
            memcpy((uint8_t*)out + (size_t)slot_bytes * r, c->h_small + (size_t)slot_bytes * r + 8, (size_t)len);
        }
        return 0;
    }, -1);
}

const char* cb200_nccl_info(void) {
    static std::string s;
    try {
        NcclApi& a = nccl();
        int v = 0;
        if (a.GetVersion) a.GetVersion(&v);
        s = "NCCL " + std::to_string(v) + " from " + a.where;
    } catch (const std::exception& e) {
        s = std::string("unavailable: ") + e.what();
    }
    return s.c_str();
}

} // extern "C"
