// vmig_common.h -- shared host-side helpers of libvmig (errors, timing, small utilities).
#pragma once
#include <stdint.h>
#include <sys/types.h>
#include <string>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cerrno>
#include <cstring>
#include "../../include/vmig.h"

namespace vmig {

// Thread-local detail of the last failure on this thread (vmig_last_error()).
void set_last_error(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
void set_last_error_str(const std::string& s);
const char* last_error_cstr();

inline uint64_t now_ns() {
    return (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
               std::chrono::steady_clock::now().time_since_epoch()).count();
}

inline int fail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
inline int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    set_last_error_str(buf);
    return code;
}

inline std::string errno_str(int e) { char b[128]; return std::string(strerror_r(e, b, sizeof b)); }

inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

// O_DIRECT file I/O needs logical-sector alignment of buffer, offset and length.
static constexpr uint32_t kSector = 4096;

// Move len bytes of a block between the file and a buffer; op(pos, n) transfers n bytes at byte pos of the block.
// direct: whole sectors (the buffer has the room), and after a short transfer the next starts at the sector boundary at
// or below what is done.  Returns 0 when len bytes are done; 1 when a call moved nothing or did not get past *done (the
// bytes done before it); else op's negative result: -1 with errno (EINTR retried when posix) or cuFile's VMIG_E* code.
template <class Op>
inline int xfer_block(bool direct, bool posix, size_t len, size_t* done, Op op)
{
    const size_t want = direct ? (size_t)align_up(len, kSector) : len;
    size_t got = 0;
    int rc = 0;
    while (got < len) {
        const size_t pos = direct ? (got & ~(size_t)(kSector - 1)) : got;
        const ssize_t r = op(pos, want - pos);
        if (r < 0 && posix && errno == EINTR) continue;
        if (r < 0) { rc = (int)r; break; }
        if (r == 0 || pos + (size_t)r <= got) { rc = 1; break; }
        got = pos + (size_t)r;
    }
    *done = got;
    return rc;
}

long env_long(const char* name, long dflt);

}  // namespace vmig
