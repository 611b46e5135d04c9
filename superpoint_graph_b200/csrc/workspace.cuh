// Scratch memory of the entry points that take a `workspace`.  One rule for all of them: the workspace is
// 256-byte aligned, every region in it starts on a 256-byte boundary, and the size its `..._workspace` query
// reports is exactly the sum of the regions.  Each stage describes its regions once, in a layout function run
// by the query with a null base (only the total is used) and by the entry points with the caller's pointer.
#pragma once
#include "common.cuh"

namespace spg {

constexpr size_t kWsAlign = 256;

// CUB's temporary storage inside a workspace; CUB's size query already covers a base of any alignment
struct CubRegion {
    void* ptr;
    size_t bytes;
};

// Bump planner: hands out consecutive regions of a workspace starting at `base`; `bytes` is the total so far.
struct Planner {
    uintptr_t base;
    size_t bytes = 0;
    explicit Planner(void* b) : base(reinterpret_cast<uintptr_t>(b)) {}
    template <class T>
    T* take(size_t n) {
        T* p = reinterpret_cast<T*>(base + bytes);
        bytes += (n * sizeof(T) + kWsAlign - 1) & ~(kWsAlign - 1);
        return p;
    }
    CubRegion cub(size_t n) { return {take<uint8_t>(n), n}; }
};

// SPG_E_BADARG for a null or short workspace, SPG_E_ALIGN for a misaligned one
inline int ws_check(const void* workspace, int64_t bytes, size_t need) {
    if (!workspace) return SPG_E_BADARG;
    if ((reinterpret_cast<uintptr_t>(workspace) & (kWsAlign - 1)) != 0) return SPG_E_ALIGN;
    return bytes < (int64_t)need ? SPG_E_BADARG : SPG_OK;
}

// counts held in int32 (CUB's item counts, indices)
inline bool too_big(int64_t n) { return n >= (1ll << 31) - 1; }

}  // namespace spg

// Raises `max_bytes` to the temporary storage CUB's `fn` needs for the remaining arguments (a size query, no
// stream); returns the query's error from the enclosing function.
#define SPG_CUB_BYTES(max_bytes, fn, ...)                                  \
    do {                                                                   \
        size_t _b = 0;                                                     \
        const cudaError_t _e = fn(nullptr, _b, __VA_ARGS__);               \
        if (_e != cudaSuccess) return (int)_e;                             \
        if (_b > (max_bytes)) (max_bytes) = _b;                            \
    } while (0)

// Runs CUB's `fn` in the CubRegion `region`; returns its error from the enclosing function.
#define SPG_CUB(region, fn, ...)                                           \
    do {                                                                   \
        size_t _b = (region).bytes;                                        \
        const cudaError_t _e = fn((region).ptr, _b, __VA_ARGS__);          \
        if (_e != cudaSuccess) return (int)_e;                             \
    } while (0)
