// bkgpu_arrow.hpp — Arrow record batches <-> bkgpu_column at the C++ host boundary (SURVEY.md §8 f2).
// The reference's vectorized engine moves fragments' inputs and results as arrow::RecordBatch (scan: RocksdbVectorizedReader::ReadNext,
// src/exec/rocksdb_scan_node.cpp:2062-2138; wire: arrow::ipc::SerializeSchema / SerializeRecordBatch into extra_res.vectorized_schema /
// vectorized_rows, src/store/region.cpp:2905-2918; db side ReadSchema / ReadRecordBatch, src/exec/fetcher_store.cpp:1130-1160).  Fields
// are named "<tuple>_<slot>" (include/expr/slot_ref.h:72-82) and typed by the Chunk map (src/runtime/chunk.cpp:33-92), which IS the
// bkgpu_column layout: fixed-width values buffer + LSB validity bitmap — so a batch enters the GPU path without a host copy.
// Needs Arrow C++ (the reference pins baikalgroup/arrow release-16.1.0; built here against pyarrow's bundled libarrow).
#pragma once
#include <arrow/api.h>
#include <arrow/io/memory.h>
#include <arrow/ipc/api.h>
#include <cstring>
#include <memory>
#include <string>
#include <vector>
#include "../include/bkgpu.h"

namespace bkgpu {

inline std::shared_ptr<arrow::DataType> arrow_type_of(int prim) {   // src/expr/arrow_function.cpp:69-96
    switch (prim) {
        case BK_BOOL: return arrow::boolean();
        case BK_INT8: case BK_INT16: case BK_INT32: case BK_TIME: return arrow::int32();
        case BK_INT64: return arrow::int64();
        case BK_UINT8: case BK_UINT16: case BK_UINT32: case BK_TIMESTAMP: case BK_DATE: return arrow::uint32();
        case BK_UINT64: case BK_DATETIME: return arrow::uint64();
        case BK_FLOAT: return arrow::float32();
        case BK_DOUBLE: return arrow::float64();
        case BK_STRING: return arrow::large_binary();
        default: return nullptr;
    }
}

// Column views over a record batch.  `declared(tuple, slot)` returns the pb::PrimitiveType the plan declares for the slot (0 = take
// the Arrow type's default: int32 -> INT32 ...).  Returns "" or an error message.  The views borrow the batch's buffers.
template <class Declared>
inline std::string columns_from_record_batch(const arrow::RecordBatch& rb, Declared declared, std::vector<bkgpu_column>* out) {
    out->clear();
    for (int i = 0; i < rb.num_columns(); i++) {
        const std::string& name = rb.schema()->field(i)->name();
        const size_t us = name.find('_');
        if (us == std::string::npos) return "field '" + name + "' is not named <tuple>_<slot>";
        bkgpu_column c{};
        c.tuple_id = std::atoi(name.substr(0, us).c_str()); c.slot_id = std::atoi(name.substr(us + 1).c_str());
        const auto& arr = rb.column(i);
        const auto& type = *arr->type();
        int prim = declared(c.tuple_id, c.slot_id), width = 0;
        switch (type.id()) {
            case arrow::Type::INT32: width = 4; if (!prim) prim = BK_INT32; break;
            case arrow::Type::UINT32: width = 4; if (!prim) prim = BK_UINT32; break;
            case arrow::Type::INT64: width = 8; if (!prim) prim = BK_INT64; break;
            case arrow::Type::UINT64: width = 8; if (!prim) prim = BK_UINT64; break;
            case arrow::Type::FLOAT: width = 4; if (!prim) prim = BK_FLOAT; break;
            case arrow::Type::DOUBLE: width = 8; if (!prim) prim = BK_DOUBLE; break;
            default: return "field '" + name + "': Arrow type " + type.ToString() + " is outside the zero-copy path";
        }
        if (!arrow_type_of(prim) || !arrow_type_of(prim)->Equals(type)) return "field '" + name + "' arrives as " + type.ToString() + " but the plan declares type " + std::to_string(prim);
        const auto& data = *arr->data();
        if (data.offset % 8 != 0 && arr->null_count() > 0) return "field '" + name + "': a sliced batch must start on a multiple of 8 rows to share its validity bitmap";
        c.prim_type = prim; c.elem_size = width; c.length = arr->length();
        c.values = data.buffers[1] ? data.buffers[1]->data() + (size_t)data.offset * (size_t)width : nullptr;
        c.validity = (arr->null_count() > 0 && data.buffers[0]) ? data.buffers[0]->data() + data.offset / 8 : nullptr;
        out->push_back(c);
    }
    return "";
}

// Result columns -> record batch with the reference's names and types (AVG intermediates as 16-byte large_binary values).
inline arrow::Result<std::shared_ptr<arrow::RecordBatch>> record_batch_from_columns(const bkgpu_column* cols, int ncols, int64_t nrows) {
    std::vector<std::shared_ptr<arrow::Field>> fields; std::vector<std::shared_ptr<arrow::Array>> arrays;
    for (int i = 0; i < ncols; i++) {
        const bkgpu_column& c = cols[i];
        if (c.prim_type == BK_BITMAP) return arrow::Status::NotImplemented("rb_build_agg's BITMAP column is not carried by the Arrow bridge");
        auto type = arrow_type_of(c.prim_type);
        if (!type) return arrow::Status::Invalid("column type outside the path");
        const std::string name = std::to_string(c.tuple_id) + "_" + std::to_string(c.slot_id);
        int64_t nulls = 0;
        std::shared_ptr<arrow::Buffer> validity;
        if (c.validity) {
            ARROW_ASSIGN_OR_RAISE(auto vb, arrow::AllocateBuffer((nrows + 7) / 8));
            std::memcpy(vb->mutable_data(), c.validity, (size_t)(nrows + 7) / 8);
            for (int64_t r = 0; r < nrows; r++) nulls += !((c.validity[r >> 3] >> (r & 7)) & 1);
            validity = std::move(vb);
        }
        std::shared_ptr<arrow::Array> arr;
        if (c.prim_type == BK_STRING) {
            arrow::LargeBinaryBuilder b;
            for (int64_t r = 0; r < nrows; r++) {
                const bool isnull = c.validity && !((c.validity[r >> 3] >> (r & 7)) & 1);
                if (isnull) ARROW_RETURN_NOT_OK(b.AppendNull()); else ARROW_RETURN_NOT_OK(b.Append((const uint8_t*)c.values + (size_t)r * 16, 16));
            }
            ARROW_RETURN_NOT_OK(b.Finish(&arr));
        } else {
            const int width = c.elem_size;
            ARROW_ASSIGN_OR_RAISE(auto vals, arrow::AllocateBuffer(nrows * width));
            if (nrows) std::memcpy(vals->mutable_data(), c.values, (size_t)nrows * (size_t)width);
            arr = arrow::MakeArray(arrow::ArrayData::Make(type, nrows, {validity, std::shared_ptr<arrow::Buffer>(std::move(vals))}, nulls));
        }
        fields.push_back(arrow::field(name, type)); arrays.push_back(arr);
    }
    return arrow::RecordBatch::Make(arrow::schema(fields), nrows, arrays);
}

// the two byte strings of the store <-> db wire
inline arrow::Status to_wire(const arrow::RecordBatch& rb, std::string* schema_bytes, std::string* rows_bytes) {
    ARROW_ASSIGN_OR_RAISE(auto s, arrow::ipc::SerializeSchema(*rb.schema()));
    ARROW_ASSIGN_OR_RAISE(auto d, arrow::ipc::SerializeRecordBatch(rb, arrow::ipc::IpcWriteOptions::Defaults()));
    schema_bytes->assign((const char*)s->data(), (size_t)s->size()); rows_bytes->assign((const char*)d->data(), (size_t)d->size());
    return arrow::Status::OK();
}
// (zero-copy: the batch aliases `rows_bytes`, which must outlive it — the reference keeps the whole response for the same reason,
//  fetcher_store.cpp:1200-1208)
inline arrow::Result<std::shared_ptr<arrow::RecordBatch>> from_wire(const std::string& schema_bytes, const std::string& rows_bytes) {
    arrow::io::BufferReader sr(std::make_shared<arrow::Buffer>((const uint8_t*)schema_bytes.data(), (int64_t)schema_bytes.size()));
    ARROW_ASSIGN_OR_RAISE(auto schema, arrow::ipc::ReadSchema(&sr, nullptr));
    arrow::io::BufferReader dr(std::make_shared<arrow::Buffer>((const uint8_t*)rows_bytes.data(), (int64_t)rows_bytes.size()));
    return arrow::ipc::ReadRecordBatch(schema, nullptr, arrow::ipc::IpcReadOptions::Defaults(), &dr);
}

}  // namespace bkgpu
