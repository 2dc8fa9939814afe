// rows.cpp -- the row primitives that hash repartitioning, Sort and HashJoin share: key kinds, uploads, column gathers and
// concatenation, packed row keys, their radix order, stable compaction and dictionary code tables.
#include "exec_internal.h"

namespace cb200 {

int key_kind(const Column& c) {
    const Phys ph = c.phys;
    switch (c.type.id) {
    case TypeId::Bool: return ph == Phys::Bitmap ? HK_BOOL : HK_BOOL8;
    case TypeId::Int8: return ph == Phys::I32 ? HK_I32 : HK_I8; // sign-extended to i32 either way
    case TypeId::Int16: return ph == Phys::I32 ? HK_I32 : HK_I16;
    case TypeId::Int32: case TypeId::Date: return HK_I32;
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: return HK_I64;
    case TypeId::Float32: return HK_F32;
    case TypeId::Float64: return HK_F64;
    case TypeId::Decimal:
        if (ph == Phys::I32) return HK_DEC_SMALL_32;
        if (ph == Phys::I64) return c.type.precision <= 18 ? HK_DEC_SMALL_64 : HK_DEC_LARGE_64;
        return c.type.precision <= 18 ? HK_DEC_SMALL_128 : HK_DEC_LARGE_128;
    case TypeId::String: case TypeId::Binary:
        if (!c.is_dict) return HK_UTF8;
        return ph == Phys::I8 ? HK_DICT8 : ph == Phys::I16 ? HK_DICT16 : HK_DICT32;
    default: throw Unsupported("hash partitioning on " + c.type.str());
    }
}

DeviceBufP host_to_device(const void* p, size_t n, ExecContext* ctx, const char* what) {
    auto b = std::make_shared<DeviceBuf>(n);
    if (n) cuda_check(cudaMemcpyAsync(b->ptr, p, n, cudaMemcpyHostToDevice, ctx->stream), what);
    cuda_check(cudaStreamSynchronize(ctx->stream), what);
    return b;
}

void columns_to_device(Batch& b, ExecContext* ctx) {
    for (auto& c : b.cols) {
        if (!c.on_host) continue;
        size_t n = (size_t)b.n_rows;
        if (c.type.is_string()) { // dictionary-encode on the host: these are group keys of a dense aggregate (a handful of rows)
            auto d = std::make_shared<Dictionary>();
            std::vector<int32_t> codes(n);
            for (size_t r = 0; r < n; r++)
                codes[r] = d->intern(std::string((const char*)c.h_data.data() + c.h_offsets[r], (size_t)(c.h_offsets[r + 1] - c.h_offsets[r])));
            c.data = host_to_device(codes.data(), n * 4, ctx, "keys H2D");
            c.is_dict = true; c.dict = d; c.phys = Phys::I32;
        } else if (c.type.id == TypeId::Bool) {
            std::vector<uint8_t> bits = pack_bits(c.h_data.data(), n);
            c.data = host_to_device(bits.data(), bits.size(), ctx, "bool H2D");
            c.phys = Phys::Bitmap;
        } else {
            c.data = host_to_device(c.h_data.data(), c.h_data.size(), ctx, "col H2D");
            c.phys = phys_of(c.type);
        }
        if (!c.h_valid.empty()) {
            std::vector<uint8_t> bits = pack_bits(c.h_valid.data(), n);
            c.validity = host_to_device(bits.data(), bits.size(), ctx, "validity H2D");
        }
        c.on_host = false;
    }
}

void arrive(Batch& b, ExecContext* ctx, const char* op) {
    columns_to_device(b, ctx);
    for (auto& c : b.cols)
        if (c.offsets) throw Unsupported(std::string(op) + " plain string columns (dictionary-encode them first)");
}

Batch drain(ExecNode& child, ExecContext* ctx, const char* op, const char* concat_op) {
    std::vector<Batch> bs;
    for (Batch in; child.next(in); in = Batch()) {
        arrive(in, ctx, op);
        if (in.n_rows > 0) bs.push_back(std::move(in));
    }
    if (bs.size() <= 1) return bs.empty() ? Batch() : std::move(bs[0]);
    return concat_batches(bs, ctx, concat_op);
}

template <typename I> void gather_columns(const Batch& in, const I* row_idx, int64_t n, Batch& out, ExecContext* ctx, const char* op) {
    cudaStream_t st = ctx->stream;
    out.n_rows = n;
    out.cols.clear();
    for (auto& c : in.cols) {
        Column o = c;
        if (c.offsets) throw Unsupported(std::string(op) + " plain string columns (dictionary-encode them first)");
        int w = phys_bytes(c.phys);
        if (w == 0) { // bit-packed booleans: gather to bytes, repack
            auto bytes = std::make_shared<DeviceBuf>((size_t)n + 16);
            launch_gather_bits(c.data->ptr, row_idx, n, bytes->ptr, st);
            ctx->kernel_launches++;
            o.data = bytes_to_bitmap(bytes, n, ctx);
            o.bool_bytes = bytes;
        } else {
            o.data = std::make_shared<DeviceBuf>((size_t)std::max<int64_t>(n, 1) * w);
            launch_gather(c.data->ptr, w, row_idx, n, o.data->ptr, st);
            ctx->kernel_launches++;
            if (c.type.id == TypeId::Bool) o.bool_bytes = o.data; // aggregate outputs keep booleans one byte per row
        }
        if (c.validity) {
            auto bytes = std::make_shared<DeviceBuf>((size_t)n + 16);
            launch_gather_bits(c.validity->ptr, row_idx, n, bytes->ptr, st);
            ctx->kernel_launches++;
            o.validity = bytes_to_bitmap(bytes, n, ctx);
            o.valid_bytes = bytes;
        }
        out.cols.push_back(o);
    }
    cuda_check(cudaGetLastError(), "gathers");
}
template void gather_columns<long long>(const Batch&, const long long*, int64_t, Batch&, ExecContext*, const char*);
template void gather_columns<unsigned>(const Batch&, const unsigned*, int64_t, Batch&, ExecContext*, const char*);

// A non-dictionary column whose batches store it in different layouts -- a Partial aggregate that migrates from dense to hash emits
// its booleans first as a bitmap (the host flush), then one byte per row (kernel output) -- is brought to the Arrow layout of its type
// in every batch first, the conversion export makes (to_arrow_layout).  Dictionary columns of different dictionaries are remapped to
// int32 codes of one new dictionary.
Batch concat_batches(const std::vector<Batch>& bs, ExecContext* ctx, const char* op) {
    cudaStream_t st = ctx->stream;
    Batch out;
    for (auto& b : bs) out.n_rows += b.n_rows;
    const size_t n = (size_t)out.n_rows;
    std::vector<DeviceBufP> temps;
    for (size_t j = 0; j < bs[0].cols.size(); j++) {
        std::vector<Column> cs;
        for (auto& b : bs) cs.push_back(b.cols[j]);
        const Column& c0 = cs[0];
        bool same = true, nulls = false;
        for (const Column& c : cs) {
            if (c.phys != c0.phys || c.dict != c0.dict || c.is_dict != c0.is_dict) same = false;
            if (c.validity) nulls = true;
        }
        if (!same && !c0.is_dict) {
            for (size_t i = 0; i < cs.size(); i++) {
                Batch one;
                one.n_rows = bs[i].n_rows;
                one.cols = {cs[i]};
                to_arrow_layout(one, ctx);
                cs[i] = one.cols[0];
                if (cs[i].phys != cs[0].phys || cs[i].is_dict) // arrive() refuses plain strings, the one type to_arrow_layout leaves alone
                    throw ExecError(15, "", std::string("internal: ") + op + " input whose batches store column " + std::to_string(j) + " in different layouts");
            }
            same = true;
        }
        Column o;
        o.type = c0.type;
        o.phys = c0.phys;
        o.is_dict = c0.is_dict;
        o.dict = c0.dict;
        if (same) {
            const int w = phys_bytes(c0.phys);
            o.data = std::make_shared<DeviceBuf>(w == 0 ? bitmap_bytes((int64_t)n) : std::max<size_t>(n, 1) * (size_t)w);
            if (w == 0) cuda_check(cudaMemsetAsync(o.data->ptr, 0, o.data->bytes, st), "memset bools");
            int64_t row = 0;
            for (size_t i = 0; i < cs.size(); i++) {
                const Batch& b = bs[i];
                const Column& c = cs[i];
                if (w == 0) { launch_bitmap_append((uint32_t*)o.data->ptr, row, (const uint8_t*)c.data->ptr, 0, b.n_rows, st); ctx->kernel_launches++; }
                else cuda_check(cudaMemcpyAsync((char*)o.data->ptr + (size_t)row * w, c.data->ptr, (size_t)b.n_rows * w, cudaMemcpyDeviceToDevice, st), "concat column");
                row += b.n_rows;
            }
        } else { // dictionary codes -> int32 codes of one dictionary
            auto d = std::make_shared<Dictionary>(*c0.dict);
            o.phys = Phys::I32;
            o.dict = d;
            o.data = std::make_shared<DeviceBuf>(std::max<size_t>(n, 1) * 4);
            int64_t row = 0;
            for (auto& b : bs) {
                const Column& c = b.cols[j];
                const std::vector<std::string>& vals = c.dict->values();
                std::vector<int32_t> table(vals.size());
                for (size_t k = 0; k < table.size(); k++) table[k] = c.dict == c0.dict ? (int32_t)k : d->intern(vals[k]);
                DeviceBufP dt = host_to_device(table.data(), table.size() * 4, ctx, "H2D remap table");
                temps.push_back(dt);
                launch_remap_codes(c.data->ptr, phys_bytes(c.phys), b.n_rows, (const int*)dt->ptr, (int)table.size(), (int*)o.data->ptr + row, st);
                ctx->kernel_launches++;
                row += b.n_rows;
            }
        }
        if (nulls) {
            o.validity = std::make_shared<DeviceBuf>(bitmap_bytes((int64_t)n));
            cuda_check(cudaMemsetAsync(o.validity->ptr, 0, o.validity->bytes, st), "memset validity");
            int64_t row = 0;
            for (auto& b : bs) {
                const Column& c = b.cols[j];
                launch_bitmap_append((uint32_t*)o.validity->ptr, row, c.validity ? (const uint8_t*)c.validity->ptr : nullptr, 0, b.n_rows, st);
                ctx->kernel_launches++;
                row += b.n_rows;
            }
            o.null_count = -1;
        }
        out.cols.push_back(o);
    }
    cuda_check(cudaGetLastError(), "concat launches");
    return out;
}

cb::SortKeyCol key_field(const Column& c, bool has_null, int& off) {
    cb::SortKeyCol f{};
    f.kind = key_kind(c);
    f.bits = sort_key_bits(c.type);
    f.data = c.data ? c.data->ptr : nullptr;
    f.validity = c.validity ? (const uint8_t*)c.validity->ptr : nullptr;
    if (c.is_dict) f.n_rank = (int)c.dict->values().size();
    f.has_null = has_null;
    f.off = off;
    off += f.bits + has_null;
    return f;
}

RowKeys pack_row_keys(const cb::SortKeyCols& kc, int64_t n, int bits, ExecContext* ctx) {
    cudaStream_t st = ctx->stream;
    const int W = kc.words;
    RowKeys rk{std::make_shared<DeviceBuf>((size_t)n * W * 8), {}, {}};
    auto and_or = std::make_shared<DeviceBuf>(2 * cb::SK_MAX_WORDS * 8);
    cuda_check(cudaMemsetAsync(and_or->ptr, 0xff, (size_t)W * 8, st), "memset key and");
    cuda_check(cudaMemsetAsync((char*)and_or->ptr + W * 8, 0, (size_t)W * 8, st), "memset key or");
    launch_sort_keys(kc, n, (unsigned long long*)rk.keys->ptr, (unsigned long long*)and_or->ptr, st);
    cuda_check(cudaGetLastError(), "k_sort_keys launch");
    ctx->kernel_launches++;
    cuda_check(cudaMemcpyAsync(rk.and_or, and_or->ptr, (size_t)W * 16, cudaMemcpyDeviceToHost, st), "D2H key and / or");
    ctx->check_device_errors(); // also synchronises
    for (int d = 0; d < (bits + 7) / 8; d++) {
        const int w = W - 1 - d / 8, sh = (d % 8) * 8;
        if (((rk.and_or[w] ^ rk.and_or[W + w]) >> sh) & 0xff) rk.digits.push_back(d);
    }
    return rk;
}

DeviceBufP radix_order(ExecContext* ctx, DeviceBufP keys0, int words, int64_t m, const std::vector<int>& digits, DeviceBufP* sorted_keys) {
    cudaStream_t st = ctx->stream;
    const int64_t nt = sort_tiles(m);
    auto keys1 = std::make_shared<DeviceBuf>((size_t)m * words * 8);
    auto idx0 = std::make_shared<DeviceBuf>((size_t)m * 4), idx1 = std::make_shared<DeviceBuf>((size_t)m * 4);
    auto hist = std::make_shared<DeviceBuf>((size_t)nt * 256 * 4), chunk_off = std::make_shared<DeviceBuf>((size_t)(nt * 256 / 4096 + 2) * 4);
    auto total = std::make_shared<DeviceBuf>(8);
    RadixScratch s{{(unsigned long long*)keys0->ptr, (unsigned long long*)keys1->ptr}, {(unsigned*)idx0->ptr, (unsigned*)idx1->ptr},
                   (unsigned*)hist->ptr, (unsigned*)chunk_off->ptr, (long long*)total->ptr};
    int r = 0;
    cuda_check(launch_sort_passes(s, words, m, digits.data(), (int)digits.size(), &r, st), "sort passes");
    ctx->kernel_launches += digits.empty() ? 1 : 4 * (int64_t)digits.size();
    if (sorted_keys) *sorted_keys = r ? keys1 : keys0;
    return r ? idx1 : idx0; // the other buffers go back to the stream-ordered pool
}

Compacted compact_rows(const DeviceBufP& keep, int64_t n, int64_t cap, ExecContext* ctx, const std::vector<std::pair<DeviceBufP, int>>& extra) {
    cudaStream_t st = ctx->stream;
    const unsigned char* flags = (const unsigned char*)keep->ptr;
    const size_t nb = (size_t)(n + 1023) / 1024;
    auto counts = std::make_shared<DeviceBuf>(nb * 4 + 4), offsets = std::make_shared<DeviceBuf>(nb * 8 + 8), kept = std::make_shared<DeviceBuf>(8);
    auto iota = std::make_shared<DeviceBuf>((size_t)n * 4);
    launch_compact_plan(flags, n, (int*)counts->ptr, (long long*)offsets->ptr, (long long*)kept->ptr, st);
    launch_sort_iota((unsigned*)iota->ptr, n, st);
    Compacted out;
    for (auto& [in, width] : extra) {
        auto o = std::make_shared<DeviceBuf>((size_t)cap * width);
        launch_compact_scatter(flags, n, (const long long*)offsets->ptr, in->ptr, width, o->ptr, st);
        out.extra_out.push_back(o);
    }
    out.rows = std::make_shared<DeviceBuf>((size_t)cap * 4);
    launch_compact_scatter(flags, n, (const long long*)offsets->ptr, iota->ptr, 4, out.rows->ptr, st);
    cuda_check(cudaGetLastError(), "compaction");
    ctx->kernel_launches += 4 + (int64_t)extra.size(); // plan (2), iota, one scatter per array
    int64_t* h_kept = (int64_t*)ctx->h_err + 1; // pinned scratch next to the error flag: both arrive after one synchronisation
    cuda_check(cudaMemcpyAsync(h_kept, kept->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H kept rows");
    ctx->check_device_errors(); // also synchronises
    out.n = *h_kept;
    return out;
}

const uint32_t* DictCodes::get(const DictionaryP& d, ExecContext* ctx, const std::function<std::vector<uint32_t>(const Dictionary&)>& make) {
    if (table && dict == d && n == d->values().size()) return (const uint32_t*)table->ptr;
    const std::vector<uint32_t> codes = make(*d);
    table = host_to_device(codes.data(), codes.size() * 4, ctx, "H2D dictionary code table");
    ctx->h2d_bytes += (int64_t)(codes.size() * 4);
    dict = d;
    n = d->values().size();
    return (const uint32_t*)table->ptr;
}

} // namespace cb200
