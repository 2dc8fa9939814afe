// proto_wire.h -- minimal protobuf wire-format reader (no protoc / libprotobuf in this image).
// Decodes the reference's prost-encoded plan IR (native/proto/src/proto/*.proto); the message
// structure lives in plan.cpp next to the field numbers it reads.
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>

namespace cb200 {

struct PbError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

struct PbReader {
    const uint8_t* p;
    const uint8_t* end;
    uint32_t field = 0;
    uint32_t wire = 0;

    PbReader(const uint8_t* data, size_t len) : p(data), end(data + len) {}

    uint64_t varint() {
        uint64_t v = 0;
        int shift = 0;
        while (true) {
            if (p >= end) throw PbError("protobuf: truncated varint");
            uint8_t b = *p++;
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) return v;
            shift += 7;
            if (shift > 63) throw PbError("protobuf: varint too long");
        }
    }
    // advance to the next field; returns false at end of message
    bool next() {
        if (p >= end) return false;
        uint64_t tag = varint();
        field = (uint32_t)(tag >> 3);
        wire = (uint32_t)(tag & 7);
        return true;
    }
    PbReader sub() { // length-delimited payload as a nested reader
        if (wire != 2) throw PbError("protobuf: expected length-delimited field");
        uint64_t n = varint();
        if ((uint64_t)(end - p) < n) throw PbError("protobuf: truncated message");
        PbReader r(p, (size_t)n);
        p += n;
        return r;
    }
    std::string bytes() {
        PbReader r = sub();
        return std::string((const char*)r.p, (size_t)(r.end - r.p));
    }
    double f64() {
        if (wire != 1 || end - p < 8) throw PbError("protobuf: bad fixed64");
        double d;
        memcpy(&d, p, 8);
        p += 8;
        return d;
    }
    float f32() {
        if (wire != 5 || end - p < 4) throw PbError("protobuf: bad fixed32");
        float f;
        memcpy(&f, p, 4);
        p += 4;
        return f;
    }
    uint32_t fixed32() { // a float's bits as sent
        if (wire != 5 || end - p < 4) throw PbError("protobuf: bad fixed32");
        uint32_t u;
        memcpy(&u, p, 4);
        p += 4;
        return u;
    }
    uint64_t fixed64() { // a double's bits as sent
        if (wire != 1 || end - p < 8) throw PbError("protobuf: bad fixed64");
        uint64_t u;
        memcpy(&u, p, 8);
        p += 8;
        return u;
    }
    int64_t i64() { // int32/int64/bool/enum fields
        if (wire != 0) throw PbError("protobuf: expected varint field");
        return (int64_t)varint();
    }
    void skip() {
        switch (wire) {
        case 0: varint(); break;
        case 1: if (end - p < 8) throw PbError("protobuf: truncated"); p += 8; break;
        case 2: sub(); break;
        case 5: if (end - p < 4) throw PbError("protobuf: truncated"); p += 4; break;
        default: throw PbError("protobuf: unsupported wire type");
        }
    }
};

} // namespace cb200
