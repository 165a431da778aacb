// table_unit.cpp -- CPU unit test of the wait before a block table that records identities is stored
// (wait_past_recorded_ctimes in csrc/vmig_table.cpp; compiled and run by tests/test_layer_versions_host.py).  A record
// trusts a file while its inode, size and ctime are unchanged.  On a kernel that stamps ctime from the coarse clock, a
// same-size write in the same tick as the record would leave all three as recorded; after the wait, a write right away
// must move the ctime whatever the kernel.  Each round records a file written just before, as a call records the files it
// has just written, and edits it in place the moment the wait returns.
//   g++ -std=c++17 -I gpu-docker-api_b200/csrc tests/table_unit.cpp gpu-docker-api_b200/csrc/vmig_table.cpp -o table_unit
#include "vmig_table.h"
#include "vmig_common.h"
#include <fcntl.h>
#include <time.h>
#include <unistd.h>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <sys/stat.h>

namespace vmig {   // the error-channel functions normally provided by vmig_engine.cu
static thread_local std::string g_err;
void set_last_error(const char* fmt, ...) { char b[1024]; va_list ap; va_start(ap, fmt); vsnprintf(b, sizeof b, fmt, ap); va_end(ap); g_err = b; }
void set_last_error_str(const std::string& s) { g_err = s; }
const char* last_error_cstr() { return g_err.c_str(); }
}
using namespace vmig;

#define CHECK(c) do { if (!(c)) { printf("FAIL line %d: %s\n", __LINE__, #c); return 1; } } while (0)

static int64_t coarse_ns() { struct timespec ts; clock_gettime(CLOCK_REALTIME_COARSE, &ts); return (int64_t)ts.tv_sec * 1000000000ll + ts.tv_nsec; }

int main(int argc, char** argv)
{
    if (argc != 2) { printf("usage: table_unit <work dir>\n"); return 2; }
    const std::string dir = argv[1];
    const std::string p = dir + "/f";
    int fd = open(p.c_str(), O_RDWR | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    CHECK(fd >= 0);
    CHECK(pwrite(fd, "0123456789abcdef", 16, 0) == 16);
    const int rounds = 200;
    for (int i = 0; i < rounds; i++) {
        const char c = (char)('A' + i % 26);
        CHECK(pwrite(fd, &c, 1, i % 16) == 1);                 // the call's own write, then its record of the file
        struct stat st;
        CHECK(fstat(fd, &st) == 0);
        BlockTable t; t.block_bytes = 4096;
        t.files.push_back({"f", (uint64_t)st.st_size, 0, (uint64_t)st.st_ino, ctime_ns(st)});
        t.files.push_back({"no_identity", 1, 1, 0, 0});          // a record without identity takes no part
        CHECK(is_recorded_file(st, t.files[0]));
        wait_past_recorded_ctimes(t);
        CHECK(coarse_ns() > t.files[0].ctime_ns);
        const char d = (char)('a' + i % 26);                    // the tenant's same-size edit, without a pause
        CHECK(pwrite(fd, &d, 1, (i + 7) % 16) == 1);
        struct stat after;
        CHECK(fstat(fd, &after) == 0);
        CHECK(after.st_ino == st.st_ino && after.st_size == st.st_size);
        CHECK(ctime_ns(after) != t.files[0].ctime_ns && ctime_ns(after) > t.files[0].ctime_ns);
        CHECK(!is_recorded_file(after, t.files[0]));
    }
    close(fd);

    // nothing to wait for: no identity at all, or a ctime far ahead of this host's clock (another host's, on a network
    // filesystem): each returns at once
    BlockTable none; none.block_bytes = 4096;
    none.files.push_back({"a", 5, 0, 0, 0});
    BlockTable ahead; ahead.block_bytes = 4096;
    ahead.files.push_back({"a", 5, 0, 42, coarse_ns() + 3600ll * 1000000000ll});
    const uint64_t t0 = now_ns();
    wait_past_recorded_ctimes(none);
    wait_past_recorded_ctimes(ahead);
    wait_past_recorded_ctimes(BlockTable());
    CHECK(now_ns() - t0 < 100000000ull);

    // a ctime within the next second is waited for, and only until the clock has passed it
    BlockTable soon; soon.block_bytes = 4096;
    const int64_t target = coarse_ns() + 30000000ll;
    soon.files.push_back({"a", 5, 0, 42, target});
    wait_past_recorded_ctimes(soon);
    const int64_t now = coarse_ns();
    CHECK(now > target && now - target < 500000000ll);
    printf("table unit ok: %d rounds\n", rounds);
    return 0;
}
