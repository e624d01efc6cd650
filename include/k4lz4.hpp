// k4lz4.hpp -- header-only C++ mirror of the reference's public block API over the C ABI
// (include/k4lz4.h).  Same names, argument meaning and error behaviour as
//   /root/reference/src/K4os.Compression.LZ4/LZ4Codec.cs:10-266, LZ4Level.cs:6-39,
//   LZ4Pickler.pickle.cs:51-106, LZ4Pickler.unpickle.cs:39-129
// for the accelerated path (L00_FAST encode, decode incl. dictionary / partial, byte[]-variant
// pickler) and Encoders/LZ4BlockEncoder.cs, LZ4BlockDecoder.cs with a batched top-up.  The reference is
// compiled managed code; with no .NET toolchain in the build image this is the compiled-language
// host side above the C ABI (INTEGRATION.md shows the C# P/Invoke stubs).
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "k4lz4.h"

namespace k4lz4 {

enum class LZ4Level : int {   // LZ4Level.cs:6-39
    L00_FAST = 0, L03_HC = 3, L04_HC = 4, L05_HC = 5, L06_HC = 6, L07_HC = 7, L08_HC = 8,
    L09_HC = 9, L10_OPT = 10, L11_OPT = 11, L12_MAX = 12
};

struct InvalidDataException : std::runtime_error { using std::runtime_error::runtime_error; };
struct NativeError : std::runtime_error {
    int code;
    NativeError(int c, const char* m) : std::runtime_error(std::string("libk4lz4: ") + m), code(c) {}
};
struct DelegateToManagedEngine : std::logic_error { using std::logic_error::logic_error; };

inline int check_codec(int r) {
    if (r <= K4LZ4_E_NODEVICE) throw NativeError(r, k4lz4_last_error());
    return r;
}

struct LZ4Codec {
    static constexpr int Version = 192;                                            // LZ4Codec.cs:13
    // LZ4Codec.Enforce32 (LZ4Codec.cs:21-25): every encode below that starts while it is set uses the 32-bit engine
    // (the k4lz4_*_x32 exports), as the reference reads its switch at each call.  Decoding is unaffected.
    static inline bool Enforce32 = false;
    static int MaximumOutputSize(int length) { return k4lz4_max_output_size(length); }   // :30-31

    // LZ4Codec.Encode(byte*,int,byte*,int,LZ4Level) -- LZ4Codec.cs:40-52
    static int Encode(const uint8_t* source, int sourceLength, uint8_t* target, int targetLength,
                      LZ4Level level = LZ4Level::L00_FAST) {
        if (sourceLength <= 0) return 0;
        const int r = check_codec((Enforce32 ? k4lz4_encode_x32 : k4lz4_encode)(source, sourceLength, target, targetLength, (int)level));
        if (r == K4LZ4_R_DELEGATE) throw DelegateToManagedEngine("HC/OPT levels stay with the managed engine");
        return r;
    }
    // LZ4Codec.Decode(byte*,int,byte*,int) -- LZ4Codec.cs:104-115
    static int Decode(const uint8_t* source, int sourceLength, uint8_t* target, int targetLength) {
        if (sourceLength <= 0) return 0;
        return check_codec(k4lz4_decode(source, sourceLength, target, targetLength));
    }
    // LZ4Codec.Decode(byte*,int,byte*,int,byte*,int) -- LZ4Codec.cs:144-157
    static int Decode(const uint8_t* source, int sourceLength, uint8_t* target, int targetLength,
                      const uint8_t* dictionary, int dictionaryLength) {
        if (sourceLength <= 0) return 0;
        return check_codec(k4lz4_decode_dict(source, sourceLength, target, targetLength, dictionary, dictionaryLength));
    }
    // LZ4Codec.PartialDecode(byte*,int,byte*,int) -- LZ4Codec.cs:123-134
    static int PartialDecode(const uint8_t* source, int sourceLength, uint8_t* target, int targetLength) {
        if (sourceLength <= 0) return 0;
        return check_codec(k4lz4_partial_decode(source, sourceLength, target, targetLength));
    }
    // The decoded length of every raw block (k4lz4_decoded_size_batch; no reference counterpart): 0 for an empty
    // block, -1 where its token chain does not parse.  Sizes the targets of Decode for blocks stored without them.
    static std::vector<int32_t> DecodedSizes(const std::vector<std::vector<uint8_t>>& blocks, int device = 0) {
        const size_t n = blocks.size();
        std::vector<int64_t> so(n);
        std::vector<int32_t> sl(n), out(n, -1);
        std::vector<uint8_t> src;
        for (size_t i = 0; i < n; i++) {
            so[i] = (int64_t)src.size(); sl[i] = (int32_t)blocks[i].size();
            src.insert(src.end(), blocks[i].begin(), blocks[i].end());
        }
        src.resize(src.size() + 1);
        const int rc = k4lz4_decoded_size_batch(src.data(), so.data(), sl.data(), out.data(), (int32_t)n,
                                                K4LZ4_MEM_HOST, nullptr, device);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        return out;
    }
};

// Independent-block stream pair with a batched top-up (SURVEY 8f row 1):
//   Encoders/LZ4EncoderBase.cs:27-97, Encoders/LZ4BlockEncoder.cs:7-23, Encoders/LZ4BlockDecoder.cs:11-102.
// Same members as the reference's ILZ4Encoder / ILZ4Decoder for one block at a time, plus
// TopupMany / EncodeMany / DecodeMany, which move a whole queue of blocks through ONE
// k4lz4_encode_batch / k4lz4_decode_batch call.  Chained (dependent-block) encoders are not data
// parallel and stay with the managed engine.
class LZ4BlockEncoder {
public:
    struct Block { int encoded; std::vector<uint8_t> bytes; };   // encoded < 0: stored raw (allowCopy)

    LZ4BlockEncoder(LZ4Level level, int blockSize, int batchBlocks = 256)
        : level_(level), block_(roundUp(blockSize < 1024 ? 1024 : blockSize, 1024)),
          depth_(batchBlocks < 1 ? 1 : batchBlocks), buf_((size_t)depth_ * block_), fill_((size_t)depth_, 0) {}

    int BlockSize() const { return block_; }
    int BytesReady() const { return cur_ < depth_ ? fill_[(size_t)cur_] : 0; }
    int BlocksQueued() const { int n = 0; for (int f : fill_) n += f > 0; return n; }

    // LZ4EncoderBase.cs:47-62
    int Topup(const uint8_t* source, int length) {
        if (length <= 0 || cur_ >= depth_) return 0;
        const int left = block_ - fill_[(size_t)cur_];
        if (left <= 0) return 0;
        const int chunk = left < length ? left : length;
        std::copy(source, source + chunk, buf_.begin() + (size_t)cur_ * block_ + fill_[(size_t)cur_]);
        fill_[(size_t)cur_] += chunk;
        return chunk;
    }
    // fills block after block until the queue or the source is exhausted
    int64_t TopupMany(const uint8_t* source, int64_t length) {
        int64_t taken = 0;
        while (taken < length && cur_ < depth_) {
            const int64_t rest = length - taken;
            const int got = Topup(source + taken, (int)(rest > block_ ? block_ : rest));
            taken += got;
            if (fill_[(size_t)cur_] == block_) cur_++;
            else if (got == 0) break;
        }
        return taken;
    }
    // LZ4EncoderBase.cs:65-87 for every queued block, one GPU call
    std::vector<Block> EncodeMany(bool allowCopy = true) {
        const int nb = BlocksQueued();
        std::vector<Block> out;
        if (nb == 0) return out;
        if ((int)level_ >= 3) throw DelegateToManagedEngine("HC/OPT levels stay with the managed engine");
        const int bound = k4lz4_max_output_size(block_);
        std::vector<int64_t> so((size_t)nb), dof((size_t)nb);
        std::vector<int32_t> sl((size_t)nb), cap((size_t)nb, bound), res((size_t)nb, -1);
        for (int i = 0; i < nb; i++) { so[(size_t)i] = (int64_t)i * block_; dof[(size_t)i] = (int64_t)i * bound; sl[(size_t)i] = fill_[(size_t)i]; }
        std::vector<uint8_t> dst((size_t)nb * bound);
        const int rc = (LZ4Codec::Enforce32 ? k4lz4_encode_batch_x32 : k4lz4_encode_batch)(buf_.data(), so.data(), sl.data(), dst.data(), dof.data(), cap.data(),
                                          res.data(), nb, (int)level_, K4LZ4_MEM_HOST, nullptr, K4LZ4_ALL_DEVICES);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        for (int i = 0; i < nb; i++) {
            const int enc = res[(size_t)i], n = sl[(size_t)i];
            if (enc <= 0) throw std::runtime_error("Failed to encode chunk. Target buffer too small.");
            Block b;
            if (allowCopy && enc >= n) { b.encoded = -n; b.bytes.assign(buf_.begin() + so[(size_t)i], buf_.begin() + so[(size_t)i] + n); }
            else { b.encoded = enc; b.bytes.assign(dst.begin() + dof[(size_t)i], dst.begin() + dof[(size_t)i] + enc); }
            out.push_back(std::move(b));
        }
        std::fill(fill_.begin(), fill_.end(), 0);        // Commit(): independent blocks keep no dictionary
        cur_ = 0;
        return out;
    }
    // the reference's single-block call
    int Encode(uint8_t* target, int length, bool allowCopy) {
        if (BlocksQueued() == 0) return 0;
        if (BlocksQueued() != 1) throw std::logic_error("Encode() handles one pending block; use EncodeMany()");
        const int n = fill_[0];
        int enc = LZ4Codec::Encode(buf_.data(), n, target, length, level_);
        if (enc <= 0) throw std::runtime_error("Failed to encode chunk. Target buffer too small.");
        if (allowCopy && enc >= n) { std::copy(buf_.begin(), buf_.begin() + n, target); enc = -n; }
        fill_[0] = 0; cur_ = 0;
        return enc;
    }

private:
    static int roundUp(int v, int step) { return (v + step - 1) / step * step; }
    LZ4Level level_;
    int block_, depth_, cur_ = 0;
    std::vector<uint8_t> buf_;
    std::vector<int> fill_;
};

class LZ4BlockDecoder {
public:
    explicit LZ4BlockDecoder(int blockSize)
        : block_(((blockSize < 1024 ? 1024 : blockSize) + 1023) / 1024 * 1024), outLen_(block_ + 8), out_((size_t)outLen_ + 8) {}
    int BlockSize() const { return block_; }
    int BytesReady() const { return index_; }
    // LZ4BlockDecoder.cs:39-55
    int Decode(const uint8_t* source, int length, int blockSize = 0) {
        if (blockSize <= 0) blockSize = block_;
        if (blockSize > block_) throw std::runtime_error("InvalidOperationException");
        const int decoded = LZ4Codec::Decode(source, length, out_.data(), outLen_);
        if (decoded < 0) throw std::runtime_error("InvalidOperationException");
        return index_ = decoded;
    }
    // one GPU call for a list of compressed blocks (raw = true: the encoder stored the block as is)
    struct Item { const uint8_t* data; int length; bool raw; };
    std::vector<std::vector<uint8_t>> DecodeMany(const std::vector<Item>& items) {
        const int n = (int)items.size();
        std::vector<std::vector<uint8_t>> res((size_t)n);
        if (n == 0) return res;
        std::vector<int64_t> so((size_t)n), dof((size_t)n);
        std::vector<int32_t> sl((size_t)n), cap((size_t)n, outLen_), got((size_t)n, -1);
        int64_t tot = 0;
        for (int i = 0; i < n; i++) { so[(size_t)i] = tot; sl[(size_t)i] = items[(size_t)i].raw ? 0 : items[(size_t)i].length; tot += sl[(size_t)i]; dof[(size_t)i] = (int64_t)i * outLen_; }
        std::vector<uint8_t> src((size_t)tot + 16), dst((size_t)n * outLen_ + 16);
        for (int i = 0; i < n; i++) if (sl[(size_t)i] > 0) std::copy(items[(size_t)i].data, items[(size_t)i].data + sl[(size_t)i], src.begin() + so[(size_t)i]);
        const int rc = k4lz4_decode_batch(src.data(), so.data(), sl.data(), dst.data(), dof.data(), cap.data(), got.data(),
                                          n, K4LZ4_MEM_HOST, nullptr, K4LZ4_ALL_DEVICES);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        for (int i = 0; i < n; i++) {
            const Item& it = items[(size_t)i];
            if (it.raw) {
                if (it.length > outLen_) throw std::runtime_error("InvalidOperationException");
                res[(size_t)i].assign(it.data, it.data + it.length);
            } else {
                if (got[(size_t)i] < 0 || (got[(size_t)i] == 0 && it.length > 0)) throw std::runtime_error("InvalidOperationException");
                res[(size_t)i].assign(dst.begin() + dof[(size_t)i], dst.begin() + dof[(size_t)i] + got[(size_t)i]);
            }
        }
        std::copy(res.back().begin(), res.back().end(), out_.begin());
        index_ = (int)res.back().size();
        return res;
    }
    // LZ4BlockDecoder.cs:58-71
    int Inject(const uint8_t* source, int length) {
        if (length <= 0) return index_ = 0;
        if (length > outLen_) throw std::runtime_error("InvalidOperationException");
        std::copy(source, source + length, out_.begin());
        return index_ = length;
    }
    // LZ4BlockDecoder.cs:74-83 (offset is negative: counted from the end of the block)
    void Drain(uint8_t* target, int offset, int length) const {
        offset = index_ + offset;
        if (offset < 0 || length < 0 || offset + length > index_) throw std::runtime_error("InvalidOperationException");
        std::copy(out_.begin() + offset, out_.begin() + offset + length, target);
    }
    const uint8_t* Peek(int offset) const {
        offset = index_ + offset;
        if (offset < 0 || offset > index_) throw std::runtime_error("InvalidOperationException");
        return out_.data() + offset;
    }

private:
    int block_, outLen_, index_ = 0;
    std::vector<uint8_t> out_;
};

// Chain groups (k4lz4_chain_group_*): S chained streams whose rings and encoder states stay on one GPU.  RAII owner
// of the group; the calls take the C ABI's batch arrays (host or device memory) and throw NativeError on a
// library-level failure.  Like the reference's encoder and decoder objects, not thread-safe.
class ChainGroup {
public:
    ChainGroup(const ChainGroup&) = delete;
    ChainGroup& operator=(const ChainGroup&) = delete;
    ChainGroup(ChainGroup&& o) noexcept : g_(o.g_) { o.g_ = nullptr; }
    ChainGroup& operator=(ChainGroup&& o) noexcept { if (this != &o) { k4lz4_chain_group_destroy(g_); g_ = o.g_; o.g_ = nullptr; } return *this; }
    ~ChainGroup() { k4lz4_chain_group_destroy(g_); }
    k4lz4_chain_group* handle() const { return g_; }
    void Reset(const int32_t* streams, int n, int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check(k4lz4_chain_group_reset(g_, streams, n, memKind, cudaStream));
    }
    // the stream's last <= 64 KiB (LZ4ChainDecoder.Peek / the encoder's dictionary)
    std::vector<uint8_t> History(int stream) const {
        std::vector<uint8_t> out(65536);
        const int k = k4lz4_chain_group_history(g_, stream, out.data(), (int)out.size());
        check(k < 0 ? k : K4LZ4_OK);
        out.resize((size_t)k);
        return out;
    }

protected:
    ChainGroup(int kind, int nStreams, int blockSize, int device) { check(k4lz4_chain_group_create(kind, nStreams, blockSize, device, &g_)); }
    static void check(int rc) { if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error()); }
    k4lz4_chain_group* g_ = nullptr;
};

class ChainEncoderGroup : public ChainGroup {
public:
    ChainEncoderGroup(int nStreams, int blockSize, int device = 0) : ChainGroup(K4LZ4_CHAIN_ENCODER, nStreams, blockSize, device) {}
    void Encode(const int32_t* streams, const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen, int n,
                LZ4Level level = LZ4Level::L00_FAST, int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check((LZ4Codec::Enforce32 ? k4lz4_chain_group_encode_x32 : k4lz4_chain_group_encode)(g_, streams, srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n,
                                       (int)level, memKind, cudaStream));
    }
    std::vector<uint8_t> State(int stream) const {
        std::vector<uint8_t> out(K4LZ4_CHAIN_STATE_BYTES);
        check(k4lz4_chain_group_state(g_, stream, out.data()));
        return out;
    }
};

class ChainDecoderGroup : public ChainGroup {
public:
    ChainDecoderGroup(int nStreams, int blockSize, int device = 0) : ChainGroup(K4LZ4_CHAIN_DECODER, nStreams, blockSize, device) {}
    void Decode(const int32_t* streams, const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen, int n,
                int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check(k4lz4_chain_group_decode(g_, streams, srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n,
                                       memKind, cudaStream));
    }
    // LZ4ChainDecoder.Inject for every listed stream
    void Inject(const int32_t* streams, const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen, int n,
                int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check(k4lz4_chain_group_inject(g_, streams, srcBase, srcOff, srcLen, n, memKind, cudaStream));
    }
};

// Frame writer groups (k4lz4_frame_writer_group_*): S LZ4EncoderStream / LZ4FrameWriter streams written
// incrementally, their partial blocks, chain states and content checksums on one GPU.  RAII owner of the group;
// Write and Close take the C ABI's arrays (host or device memory) and append to each entry's destination.
// flags: K4LZ4_FRAME_*.  A level >= 3 throws DelegateToManagedEngine.  Not thread-safe.
class FrameWriterGroup {
public:
    FrameWriterGroup(int nStreams, int blockSize = 65536, int flags = 0, LZ4Level level = LZ4Level::L00_FAST,
                     int device = 0) {
        const int rc = k4lz4_frame_writer_group_create(nStreams, blockSize, flags, (int)level, device, &g_);
        if (rc == K4LZ4_R_DELEGATE) throw DelegateToManagedEngine("chained HC levels stay with the managed engine");
        check(rc);
    }
    FrameWriterGroup(const FrameWriterGroup&) = delete;
    FrameWriterGroup& operator=(const FrameWriterGroup&) = delete;
    FrameWriterGroup(FrameWriterGroup&& o) noexcept : g_(o.g_) { o.g_ = nullptr; }
    FrameWriterGroup& operator=(FrameWriterGroup&& o) noexcept {
        if (this != &o) { k4lz4_frame_writer_group_destroy(g_); g_ = o.g_; o.g_ = nullptr; }
        return *this;
    }
    ~FrameWriterGroup() { k4lz4_frame_writer_group_destroy(g_); }
    k4lz4_frame_writer_group* handle() const { return g_; }
    int64_t Bound(int64_t length) const { return k4lz4_frame_writer_bound(g_, length); }
    int64_t CloseBound() const { return k4lz4_frame_writer_close_bound(g_); }
    void Write(const int32_t* streams, const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
               uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen, int n,
               int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check((LZ4Codec::Enforce32 ? k4lz4_frame_writer_group_write_x32 : k4lz4_frame_writer_group_write)(g_, streams, srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n,
                                             memKind, cudaStream));
    }
    void Close(const int32_t* streams, uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen,
               int n, int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check((LZ4Codec::Enforce32 ? k4lz4_frame_writer_group_close_x32 : k4lz4_frame_writer_group_close)(g_, streams, dstBase, dstOff, dstCap, outLen, n, memKind, cudaStream));
    }
    void Reset(const int32_t* streams, int n, int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check(k4lz4_frame_writer_group_reset(g_, streams, n, memKind, cudaStream));
    }

private:
    static void check(int rc) { if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error()); }
    k4lz4_frame_writer_group* g_ = nullptr;
};

// LZ4DecoderStream / LZ4FrameReader for many streams (k4lz4.h "frame reader group"); move-only.
class FrameReaderGroup {
public:
    explicit FrameReaderGroup(int nStreams, int maxBlockSize = 65536, int device = 0) {
        check(k4lz4_frame_reader_group_create(nStreams, maxBlockSize, device, &g_));
    }
    FrameReaderGroup(const FrameReaderGroup&) = delete;
    FrameReaderGroup& operator=(const FrameReaderGroup&) = delete;
    FrameReaderGroup(FrameReaderGroup&& o) noexcept : g_(o.g_) { o.g_ = nullptr; }
    FrameReaderGroup& operator=(FrameReaderGroup&& o) noexcept {
        if (this != &o) { k4lz4_frame_reader_group_destroy(g_); g_ = o.g_; o.g_ = nullptr; }
        return *this;
    }
    ~FrameReaderGroup() { k4lz4_frame_reader_group_destroy(g_); }
    k4lz4_frame_reader_group* handle() const { return g_; }
    void Read(const int32_t* streams, const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
              int32_t* srcUsed, uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen,
              int32_t* frameEnded, int n, int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check(k4lz4_frame_reader_group_read(g_, streams, srcBase, srcOff, srcLen, srcUsed, dstBase, dstOff, dstCap,
                                            outLen, frameEnded, n, memKind, cudaStream));
    }
    // Destinations of any size: drains the current block first, keeps what does not fit for the next call.
    void ReadBytes(const int32_t* streams, const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                   int32_t* srcUsed, uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen,
                   int32_t* frameEnded, int n, bool interactive = false, int memKind = K4LZ4_MEM_HOST,
                   void* cudaStream = nullptr) {
        check(k4lz4_frame_reader_group_read_bytes(g_, streams, srcBase, srcOff, srcLen, srcUsed, dstBase, dstOff,
                                                  dstCap, outLen, frameEnded, n,
                                                  interactive ? K4LZ4_READ_INTERACTIVE : 0, memKind, cudaStream));
    }
    void End(const int32_t* streams, int32_t* status, int n, int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check(k4lz4_frame_reader_group_end(g_, streams, status, n, memKind, cudaStream));
    }
    void Reset(const int32_t* streams, int n, int memKind = K4LZ4_MEM_HOST, void* cudaStream = nullptr) {
        check(k4lz4_frame_reader_group_reset(g_, streams, n, memKind, cudaStream));
    }

private:
    static void check(int rc) { if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error()); }
    k4lz4_frame_reader_group* g_ = nullptr;
};

struct LZ4Pickler {
    // LZ4Pickler.Pickle(ReadOnlySpan<byte>, LZ4Level) -- LZ4Pickler.pickle.cs:51-74
    static std::vector<uint8_t> Pickle(const uint8_t* source, int length, LZ4Level level = LZ4Level::L00_FAST) {
        if (length == 0) return {};
        std::vector<uint8_t> out((size_t)k4lz4_pickle_bound(length));
        int64_t so = 0, dof = 0; int32_t n = length, r = -1;
        const int rc = (LZ4Codec::Enforce32 ? k4lz4_pickle_batch_x32 : k4lz4_pickle_batch)(source, &so, &n, out.data(), &dof, &r, 1, (int)level, K4LZ4_MEM_HOST, nullptr, 0);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        if (r == K4LZ4_R_DELEGATE) throw DelegateToManagedEngine("HC/OPT levels stay with the managed engine");
        out.resize((size_t)r);
        return out;
    }
    // LZ4Pickler.UnpickledSize -- LZ4Pickler.unpickle.cs:83-92
    static int UnpickledSize(const uint8_t* source, int length) {
        int64_t so = 0; int32_t n = length, r = -1;
        const int rc = k4lz4_unpickled_size_batch(source, &so, &n, &r, 1, K4LZ4_MEM_HOST, nullptr, 0);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        if (r == K4LZ4_R_CORRUPT) throw InvalidDataException("Pickle is corrupted");
        return r;
    }
    // LZ4Pickler.Unpickle(ReadOnlySpan<byte>) -- LZ4Pickler.unpickle.cs:39-50
    static std::vector<uint8_t> Unpickle(const uint8_t* source, int length) {
        if (length == 0) return {};
        const int size = UnpickledSize(source, length);
        std::vector<uint8_t> out((size_t)size);
        if (size == 0) return out;
        int64_t so = 0, dof = 0; int32_t n = length, dl = size, r = -1;
        const int rc = k4lz4_unpickle_batch(source, &so, &n, out.data(), &dof, &dl, &r, 1, K4LZ4_MEM_HOST, nullptr, 0);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        if (r == K4LZ4_R_CORRUPT) throw InvalidDataException("Pickle is corrupted");
        return out;
    }
};

// LZ4Frame.Encode / Decode over whole buffers (k4lz4_frame_*): one frame, or many in one call (host memory).
struct LZ4FrameSettings {      // LZ4EncoderSettings: the reference's defaults
    int blockSize = 65536;
    bool chainBlocks = true, blockChecksum = false, contentChecksum = false;
    LZ4Level level = LZ4Level::L00_FAST;
};

struct LZ4Frame {
    using Settings = LZ4FrameSettings;
    static int flags(const Settings& s) {
        return (s.chainBlocks ? 0 : K4LZ4_FRAME_INDEPENDENT) | (s.blockChecksum ? K4LZ4_FRAME_BLOCK_CHECKSUM : 0) |
               (s.contentChecksum ? K4LZ4_FRAME_CONTENT_CHECKSUM : 0);
    }
    static int64_t Bound(int64_t length, const Settings& s = {}) {
        const int64_t r = k4lz4_frame_bound(length, s.blockSize, flags(s));
        if (r < 0) throw NativeError((int)r, k4lz4_last_error());
        return r;
    }
    // frame i of the result holds sources[i]
    static std::vector<std::vector<uint8_t>> EncodeMany(const std::vector<std::vector<uint8_t>>& sources,
                                                        const Settings& s = {}, int device = 0) {
        const size_t n = sources.size();
        std::vector<int64_t> so(n), dofs(n);
        std::vector<int32_t> sl(n), dc(n), out(n, -1);
        std::vector<uint8_t> src, dst;
        int64_t d = 0;
        for (size_t i = 0; i < n; i++) {
            so[i] = (int64_t)src.size(); sl[i] = (int32_t)sources[i].size();
            src.insert(src.end(), sources[i].begin(), sources[i].end());
            dofs[i] = d; dc[i] = (int32_t)Bound(sl[i], s); d += dc[i];
        }
        src.resize(src.size() + 1); dst.resize((size_t)d + 1);
        const int rc = (LZ4Codec::Enforce32 ? k4lz4_frame_encode_batch_x32 : k4lz4_frame_encode_batch)(src.data(), so.data(), sl.data(), dst.data(), dofs.data(), dc.data(),
                                                out.data(), (int32_t)n, s.blockSize, flags(s), (int)s.level,
                                                K4LZ4_MEM_HOST, nullptr, device);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        std::vector<std::vector<uint8_t>> frames(n);
        for (size_t i = 0; i < n; i++) {
            if (out[i] == K4LZ4_R_DELEGATE) throw DelegateToManagedEngine("chained HC levels stay managed");
            if (out[i] < 0) throw std::runtime_error("Failed to encode chunk. Target buffer too small.");
            frames[i].assign(dst.begin() + dofs[i], dst.begin() + dofs[i] + out[i]);
        }
        return frames;
    }
    static std::vector<uint8_t> Encode(const std::vector<uint8_t>& source, const Settings& s = {}, int device = 0) {
        return EncodeMany({source}, s, device)[0];
    }
    static std::vector<int32_t> ContentSizes(const std::vector<std::vector<uint8_t>>& frames, int device = 0) {
        const size_t n = frames.size();
        std::vector<int64_t> so(n);
        std::vector<int32_t> sl(n), out(n, -1);
        std::vector<uint8_t> src;
        for (size_t i = 0; i < n; i++) {
            so[i] = (int64_t)src.size(); sl[i] = (int32_t)frames[i].size();
            src.insert(src.end(), frames[i].begin(), frames[i].end());
        }
        src.resize(src.size() + 1);
        const int rc = k4lz4_frame_content_size_batch(src.data(), so.data(), sl.data(), out.data(), (int32_t)n,
                                                      K4LZ4_MEM_HOST, nullptr, device);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        return out;
    }
    static int64_t ContentSize(const std::vector<uint8_t>& frame, int device = 0) {
        const int32_t r = ContentSizes({frame}, device)[0];
        raise_for(r);
        return r;
    }
    static std::vector<std::vector<uint8_t>> DecodeMany(const std::vector<std::vector<uint8_t>>& frames, int device = 0) {
        const size_t n = frames.size();
        const std::vector<int32_t> sizes = ContentSizes(frames, device);
        std::vector<int64_t> so(n), dofs(n);
        std::vector<int32_t> sl(n), dc(n), out(n, -1);
        std::vector<uint8_t> src, dst;
        int64_t d = 0;
        for (size_t i = 0; i < n; i++) {
            so[i] = (int64_t)src.size(); sl[i] = (int32_t)frames[i].size();
            src.insert(src.end(), frames[i].begin(), frames[i].end());
            dofs[i] = d; dc[i] = std::max<int32_t>(sizes[i], 0); d += dc[i];
        }
        src.resize(src.size() + 1); dst.resize((size_t)d + 1);
        const int rc = k4lz4_frame_decode_batch(src.data(), so.data(), sl.data(), dst.data(), dofs.data(), dc.data(),
                                                out.data(), (int32_t)n, K4LZ4_MEM_HOST, nullptr, device);
        if (rc != K4LZ4_OK) throw NativeError(rc, k4lz4_last_error());
        std::vector<std::vector<uint8_t>> contents(n);
        for (size_t i = 0; i < n; i++) {
            raise_for(out[i]);
            contents[i].assign(dst.begin() + dofs[i], dst.begin() + dofs[i] + out[i]);
        }
        return contents;
    }
    static std::vector<uint8_t> Decode(const std::vector<uint8_t>& frame, int device = 0) {
        return DecodeMany({frame}, device)[0];
    }
private:
    static void raise_for(int32_t r) {
        if (r == K4LZ4_R_DELEGATE) throw DelegateToManagedEngine("Predefined dictionaries feature is not implemented");
        if (r < 0) throw InvalidDataException("Invalid LZ4 frame");
    }
};

}  // namespace k4lz4
