// Context, memory, timing and the scratch arena of liburh_b200.
#include "common.cuh"
#include "tilescan.cuh"

extern "C" int urh_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

extern "C" int urh_ctx_create(int device, urh_ctx** out) {
    if (!out) return URH_ERR_INVALID;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return URH_ERR_NO_DEVICE;
    if (device < 0 || device >= n) return URH_ERR_INVALID;
    urh_ctx* ctx = new urh_ctx();
    ctx->device = device;
    ctx->err[0] = 0;
    ctx->launches = 0;
    ctx->arena_block = 0;
    ctx->arena_used = 0;
    ctx->arena_need = 0;
    ctx->pulses = nullptr;
    ctx->pulses_cap_rows = 0;
    ctx->pulses_k = 0;
    ctx->h_mail = nullptr;
    ctx->h_stage[0] = ctx->h_stage[1] = nullptr;
    ctx->h_stage_bytes = 0;
    ctx->fft_valid = false;
    ctx->shard_state = nullptr;
    ctx->costas_shard = nullptr;
    ctx->bits_valid = 0;
    ctx->mod_plan_valid[0] = ctx->mod_plan_valid[1] = 0;
    ctx->center_prefix = nullptr;
    ctx->center_ts = nullptr;
    ctx->center_x = nullptr;
    ctx->center_n = 0;
    ctx->nccl_comm = nullptr;
    ctx->nccl_stage = nullptr;
    ctx->nccl_hstage = nullptr;
    ctx->nccl_rank = 0;
    ctx->nccl_world = 1;
    ctx->stream_free_low = -1;
    ctx->stream_chunks = 0;
    if (cudaSetDevice(device) != cudaSuccess) {
        delete ctx;
        return URH_ERR_CUDA;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
        delete ctx;
        return URH_ERR_CUDA;
    }
    ctx->sm_count = prop.multiProcessorCount;
    {
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
            unsigned long long keep = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
    }
    bool ok = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&ctx->copy_stream[0], cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&ctx->copy_stream[1], cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreate(&ctx->ev_start) == cudaSuccess && cudaEventCreate(&ctx->ev_stop) == cudaSuccess;
    for (int i = 0; i < 2 && ok; i++) {
        ok = ok && cudaEventCreateWithFlags(&ctx->ev_copy[i], cudaEventDisableTiming) == cudaSuccess;
        ok = ok && cudaEventCreateWithFlags(&ctx->ev_comp[i], cudaEventDisableTiming) == cudaSuccess;
    }
    ok = ok && cudaEventCreate(&ctx->ev_k0) == cudaSuccess && cudaEventCreate(&ctx->ev_k1) == cudaSuccess;
    ctx->profiling = 0;
    ctx->dense_timed = 0;
    ctx->tl_count = 0;
    ctx->tl_ready = 0;
    ok = ok && cudaHostAlloc((void**)&ctx->h_mail, 64 * sizeof(int64_t), cudaHostAllocDefault) == cudaSuccess;
    if (!ok) {
        delete ctx;
        return URH_ERR_CUDA;
    }
    *out = ctx;
    return URH_OK;
}

extern "C" void urh_ctx_destroy(urh_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    urh_release_mod_plans(ctx);
    for (auto& b : ctx->arena) cudaFree(b.ptr);
    if (ctx->pulses) cudaFree(ctx->pulses);
    if (ctx->shard_state) free(ctx->shard_state);
    urh_costas_shard_release(ctx);
    if (ctx->h_mail) cudaFreeHost(ctx->h_mail);
    if (ctx->ts_mem) cudaFree(ctx->ts_mem);
    if (ctx->step_dev) cudaFree(ctx->step_dev);
    if (ctx->img_tw) cudaFree(ctx->img_tw);
    if (ctx->shard_fin) free(ctx->shard_fin);
    for (int i = 0; i < 2; i++)
        if (ctx->h_stage[i]) cudaFreeHost(ctx->h_stage[i]);
    cudaEventDestroy(ctx->ev_start);
    cudaEventDestroy(ctx->ev_stop);
    for (int i = 0; i < 2; i++) {
        cudaEventDestroy(ctx->ev_copy[i]);
        cudaEventDestroy(ctx->ev_comp[i]);
        cudaStreamDestroy(ctx->copy_stream[i]);
    }
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

extern "C" const char* urh_last_error(urh_ctx* ctx) { return ctx ? ctx->err : "null context"; }

extern "C" int urh_sync(urh_ctx* ctx) {
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

extern "C" int urh_device_info(urh_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem,
                               char* name, int name_cap) {
    cudaDeviceProp prop;
    URH_CUDA(ctx, cudaGetDeviceProperties(&prop, ctx->device));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    if (total_mem) *total_mem = prop.totalGlobalMem;
    if (name && name_cap > 0) {
        strncpy(name, prop.name, name_cap - 1);
        name[name_cap - 1] = 0;
    }
    return URH_OK;
}

// Stream-ordered allocation from the device's default memory pool (release threshold = never, set in
// urh_ctx_create): the result arrays of repeated calls come back in microseconds instead of cudaMalloc's milliseconds.
extern "C" int urh_malloc(urh_ctx* ctx, size_t bytes, void** d_ptr) {
    URH_CUDA(ctx, cudaSetDevice(ctx->device));
    if (bytes == 0) bytes = 16;
    URH_CUDA(ctx, cudaMallocAsync(d_ptr, bytes, ctx->stream));
    return URH_OK;
}

extern "C" int urh_free(urh_ctx* ctx, void* d_ptr) {
    if (!d_ptr) return URH_OK;
    URH_CUDA(ctx, cudaFreeAsync(d_ptr, ctx->stream));
    return URH_OK;
}

extern "C" int urh_memset(urh_ctx* ctx, void* d_ptr, int value, size_t bytes) {
    URH_CUDA(ctx, cudaMemsetAsync(d_ptr, value, bytes, ctx->stream));
    return URH_OK;
}

extern "C" int urh_memcpy_h2d(urh_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
    if (bytes == 0) return URH_OK;
    URH_CUDA(ctx, cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return URH_OK;
}

extern "C" int urh_memcpy_d2h(urh_ctx* ctx, void* h_dst, const void* d_src, size_t bytes) {
    if (bytes) URH_CUDA(ctx, cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

extern "C" int urh_memcpy_d2d(urh_ctx* ctx, void* d_dst, const void* d_src, size_t bytes) {
    if (bytes == 0) return URH_OK;
    URH_CUDA(ctx, cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return URH_OK;
}

extern "C" int urh_host_alloc(urh_ctx* ctx, size_t bytes, void** h_ptr) {
    if (bytes == 0) bytes = 16;
    URH_CUDA(ctx, cudaHostAlloc(h_ptr, bytes, cudaHostAllocDefault));
    return URH_OK;
}

extern "C" int urh_host_free(urh_ctx* ctx, void* h_ptr) {
    if (h_ptr) URH_CUDA(ctx, cudaFreeHost(h_ptr));
    return URH_OK;
}

extern "C" int urh_timer_start(urh_ctx* ctx) {
    URH_CUDA(ctx, cudaEventRecord(ctx->ev_start, ctx->stream));
    return URH_OK;
}

extern "C" int urh_timer_stop(urh_ctx* ctx, float* ms) {
    URH_CUDA(ctx, cudaEventRecord(ctx->ev_stop, ctx->stream));
    URH_CUDA(ctx, cudaEventSynchronize(ctx->ev_stop));
    float t = 0.f;
    URH_CUDA(ctx, cudaEventElapsedTime(&t, ctx->ev_start, ctx->ev_stop));
    if (ms) *ms = t;
    return URH_OK;
}

extern "C" int urh_set_profiling(urh_ctx* ctx, int enabled) {
    ctx->profiling = enabled < 0 ? 0 : (enabled > 2 ? 2 : enabled);
    ctx->dense_timed = 0;
    if (ctx->profiling >= 2 && !ctx->tl_ready) {
        for (int i = 0; i < 32; i++) URH_CUDA(ctx, cudaEventCreate(&ctx->tl_ev[i]));
        ctx->tl_ready = 1;
    }
    ctx->tl_count = 0;
    return URH_OK;
}

// Timeline of the last sharded step (profiling level 2): milliseconds from the step's first mark to each mark, and the marks' names
// ('\n'-separated, into h_names).  Call after the step's result has been read (the stream is idle).
extern "C" int urh_timeline_fetch(urh_ctx* ctx, float* h_ms, char* h_names, int names_cap, int* count) {
    if (!count) return URH_ERR_INVALID;
    *count = 0;
    if (ctx->profiling < 2 || ctx->tl_count == 0) return URH_OK;
    URH_CUDA(ctx, cudaEventSynchronize(ctx->tl_ev[ctx->tl_count - 1]));
    int pos = 0;
    for (int i = 0; i < ctx->tl_count; i++) {
        float t = 0.f;
        URH_CUDA(ctx, cudaEventElapsedTime(&t, ctx->tl_ev[0], ctx->tl_ev[i]));
        if (h_ms) h_ms[i] = t;
        if (h_names) pos += snprintf(h_names + pos, pos < names_cap ? (size_t)(names_cap - pos) : 0, "%s\n", ctx->tl_name[i]);
    }
    *count = ctx->tl_count;
    return URH_OK;
}

extern "C" int urh_last_dense_ms(urh_ctx* ctx, float* ms) {
    if (!ctx->dense_timed) URH_FAIL(ctx, URH_ERR_INVALID, "no dense kernel timed (enable urh_set_profiling first)");
    URH_CUDA(ctx, cudaEventSynchronize(ctx->ev_k1));
    URH_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev_k0, ctx->ev_k1));
    return URH_OK;
}

extern "C" int64_t urh_launch_count(urh_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ---- arena ----------------------------------------------------------------------------------------
// Kernels enqueued earlier may still be reading arena memory when the next op resets the bump pointer;
// all ops run on the one ctx stream, so reuse is stream-ordered and safe.  Growing (cudaFree) needs a sync.
void urh_arena_reset(urh_ctx* ctx) {
    if (ctx->arena.size() > 1) {
        // coalesce into one block big enough for everything the last op asked for
        cudaStreamSynchronize(ctx->stream);
        size_t total = 0;
        for (auto& b : ctx->arena) {
            total += b.bytes;
            cudaFree(b.ptr);
        }
        ctx->arena.clear();
        void* p = nullptr;
        if (cudaMalloc(&p, total) == cudaSuccess) ctx->arena.push_back({p, total});
        else cudaGetLastError();
    }
    ctx->arena_block = 0;
    ctx->arena_used = 0;
    ctx->arena_need = 0;
    ctx->arena_live = 0;
    ctx->arena_peak = 0;
    ctx->center_prefix = nullptr;  // the detect_center tile table lived in the arena
    ctx->bits_valid = 0;           // so did the bit arrays
}

static void arena_note_peak(urh_ctx* ctx) {
    if (ctx->arena_live > ctx->arena_peak) ctx->arena_peak = ctx->arena_live;
}

int urh_arena_alloc(urh_ctx* ctx, size_t bytes, void** out) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (bytes == 0) bytes = 256;
    ctx->arena_need += bytes;
    ctx->arena_live += bytes;
    while (ctx->arena_block < ctx->arena.size()) {
        urh_block& b = ctx->arena[ctx->arena_block];
        if (ctx->arena_used + bytes <= b.bytes) {
            *out = (char*)b.ptr + ctx->arena_used;
            ctx->arena_used += bytes;
            arena_note_peak(ctx);
            return URH_OK;
        }
        ctx->arena_block++;
        ctx->arena_used = 0;
    }
    size_t want = bytes > ((size_t)64 << 20) ? bytes : ((size_t)64 << 20);
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess && want > bytes) {
        cudaGetLastError();
        want = bytes;
        e = cudaMalloc(&p, want);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        snprintf(ctx->err, sizeof(ctx->err), "arena: cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
        return URH_ERR_NOMEM;
    }
    ctx->arena.push_back({p, want});
    ctx->arena_block = ctx->arena.size() - 1;
    ctx->arena_used = bytes;
    arena_note_peak(ctx);
    *out = p;
    return URH_OK;
}

int urh_ensure_pulses(urh_ctx* ctx, size_t rows) {
    if (rows < 16) rows = 16;
    if (rows <= ctx->pulses_cap_rows) return URH_OK;
    if (ctx->pulses) {
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        URH_CUDA(ctx, cudaFree(ctx->pulses));
        ctx->pulses = nullptr;
        ctx->pulses_cap_rows = 0;
    }
    size_t cap = rows + rows / 4;
    URH_CUDA(ctx, cudaMalloc((void**)&ctx->pulses, cap * 2 * sizeof(int64_t)));
    ctx->pulses_cap_rows = cap;
    return URH_OK;
}

int urh_ensure_pulses_keep(urh_ctx* ctx, size_t rows, size_t keep) {
    if (rows <= ctx->pulses_cap_rows) return URH_OK;
    int64_t* p = nullptr;
    URH_CUDA(ctx, cudaMalloc((void**)&p, rows * 2 * sizeof(int64_t)));
    urh_stream_sample_free(ctx);   // the old and the new table coexist here
    if (ctx->pulses) {
        if (keep) URH_CUDA(ctx, cudaMemcpyAsync(p, ctx->pulses, keep * 2 * sizeof(int64_t), cudaMemcpyDeviceToDevice, ctx->stream));
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        URH_CUDA(ctx, cudaFree(ctx->pulses));
    }
    ctx->pulses = p;
    ctx->pulses_cap_rows = rows;
    return URH_OK;
}

void urh_stream_sample_free(urh_ctx* ctx) {
    if (!ctx->profiling) return;   // a driver call per chunk: only when measuring
    size_t fr = 0, tot = 0;
    if (cudaMemGetInfo(&fr, &tot) == cudaSuccess && (ctx->stream_free_low < 0 || (int64_t)fr < ctx->stream_free_low))
        ctx->stream_free_low = (int64_t)fr;
}

extern "C" int urh_mem_get_info(urh_ctx* ctx, size_t* free_bytes, size_t* total_bytes) {
    URH_CUDA(ctx, cudaSetDevice(ctx->device));
    URH_CUDA(ctx, cudaMemGetInfo(free_bytes, total_bytes));
    return URH_OK;
}

// Workspace of the look-back scans (tilescan.cuh): [counter 256 B][status 4 B x cap][agg SLOT x cap][pre SLOT x cap].
// Zeroed once; launches are told apart by their epoch and by the counter value their first block will draw.
int urhts::prepare(urh_ctx* ctx, int64_t nblocks, urhts::Ws* out) {
    if (nblocks > ctx->ts_cap_blocks) {
        if (ctx->ts_mem) {
            URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            URH_CUDA(ctx, cudaFree(ctx->ts_mem));
            ctx->ts_mem = nullptr;
            ctx->ts_cap_blocks = 0;
        }
        int64_t cap = nblocks * 2 > 8192 ? nblocks * 2 : 8192;
        cap = (cap + 63) & ~(int64_t)63;
        const size_t bytes = 256 + (size_t)cap * (4 + 2 * urhts::SLOT);
        URH_CUDA(ctx, cudaMalloc(&ctx->ts_mem, bytes));
        URH_CUDA(ctx, cudaMemsetAsync(ctx->ts_mem, 0, bytes, ctx->stream));
        ctx->ts_cap_blocks = cap;
        ctx->ts_issued = 0;
        ctx->ts_epoch = 0;
    }
    char* base = (char*)ctx->ts_mem;
    out->counter = (unsigned long long*)base;
    out->status = (uint32_t*)(base + 256);
    out->agg = base + 256 + (size_t)ctx->ts_cap_blocks * 4;
    out->pre = out->agg + (size_t)ctx->ts_cap_blocks * urhts::SLOT;
    out->base = ctx->ts_issued;
    ctx->ts_issued += (unsigned long long)nblocks;
    ctx->ts_epoch = (ctx->ts_epoch + 1) & 0x3fffffffu;
    if (ctx->ts_epoch == 0) ctx->ts_epoch = 1;   // 0 is the zero-initialised "never written" state
    out->epoch = ctx->ts_epoch;
    return URH_OK;
}

int urh_ensure_stage(urh_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->h_stage_bytes) return URH_OK;
    for (int i = 0; i < 2; i++) {
        if (ctx->h_stage[i]) URH_CUDA(ctx, cudaFreeHost(ctx->h_stage[i]));
        ctx->h_stage[i] = nullptr;
    }
    ctx->h_stage_bytes = 0;
    for (int i = 0; i < 2; i++) URH_CUDA(ctx, cudaHostAlloc(&ctx->h_stage[i], bytes, cudaHostAllocDefault));
    ctx->h_stage_bytes = bytes;
    return URH_OK;
}

int urh_read_i64(urh_ctx* ctx, const int64_t* d_src, int count, int64_t* h_out) {
    if (count > 64) return URH_ERR_INVALID;
    URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail, d_src, count * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < count; i++) h_out[i] = ctx->h_mail[i];
    return URH_OK;
}
