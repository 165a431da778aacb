// prefault_probe.cpp -- host measurement (not part of libvmig; no GPU): can the pwrite streams that fill NEW tmpfs files
// be made cheaper by allocating their pages ahead of them on other threads, the way libvmig's readers would?  Ten
// 1 GiB files, one pwrite stream each (4 MiB chunks); five more threads allocate chunk k of file f before its writer
// reaches it, either by madvise(MADV_POPULATE_WRITE) through a shared mapping (the fault path: no inode lock on Linux
// >= 5.14) or by fallocate.  Every variant runs twice: a second pass reuses the memory the first one freed.
//   g++ -O2 -pthread -o prefault_probe prefault_probe.cpp ; ./prefault_probe /dev/shm/vmig_pfprobe
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <atomic>
#include <cerrno>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>
#ifndef MADV_POPULATE_WRITE
#define MADV_POPULATE_WRITE 23
#endif
static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static void par(int T, const std::function<void(int)>& f) { std::vector<std::thread> th; for (int t = 0; t < T; t++) th.emplace_back(f, t); for (auto& x : th) x.join(); }
int main(int argc, char** argv) {
    std::string dir = argc > 1 ? argv[1] : "/dev/shm/vmig_pfprobe";
    mkdir(dir.c_str(), 0755);
    const size_t G = 1ull << 30, CH = 4 << 20, SB = 256 << 20; const int F = 10;
    char* src = (char*)aligned_alloc(4096, SB); memset(src, 7, SB);
    auto path = [&](int i) { return dir + "/f" + std::to_string(i); };
    auto cleanup = [&] { for (int f = 0; f < F; f++) unlink(path(f).c_str()); };
    {   // does the kernel have the advice, and what does it cost on one thread?
        int fd = open(path(0).c_str(), O_RDWR | O_CREAT | O_TRUNC, 0644); if (ftruncate(fd, G)) perror("ftruncate");
        char* m = (char*)mmap(0, G, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        double t0 = now(); int r = madvise(m, G, MADV_POPULATE_WRITE); int e = errno; double dt = now() - t0;
        printf("madvise(MADV_POPULATE_WRITE, 1 GiB): %s", r ? strerror(e) : "ok");
        if (!r) printf(", %.2f GB/s", G / dt / 1e9);
        printf("\n");
        munmap(m, G); close(fd); cleanup();
    }
    for (int mode = 0; mode < 3; mode++)
        for (int rep = 0; rep < 2; rep++) {
            // 0: writers alone; 1: five threads MADV_POPULATE_WRITE ahead; 2: five threads fallocate ahead
            std::vector<int> fds(F); std::vector<char*> maps(F, nullptr);
            std::vector<std::atomic<size_t>> ready(F);
            double t0 = now();
            for (int f = 0; f < F; f++) {
                fds[f] = open(path(f).c_str(), O_RDWR | O_CREAT | O_TRUNC, 0644); ready[f] = mode ? 0 : G;
                if (mode == 1) { if (ftruncate(fds[f], G)) perror("ftruncate"); maps[f] = (char*)mmap(0, G, PROT_READ | PROT_WRITE, MAP_SHARED, fds[f], 0); }
            }
            std::atomic<size_t> next{0}; const size_t total = F * (G / CH);
            std::atomic<int> failed{0};
            std::thread pool([&] { if (mode) par(5, [&](int) { for (;;) {
                size_t k = next.fetch_add(1); if (k >= total) break;
                const int f = k % F; const size_t o = (k / F) * CH;
                if ((mode == 1 ? madvise(maps[f] + o, CH, MADV_POPULATE_WRITE) : fallocate(fds[f], 0, o, CH)) != 0) failed++;
                size_t want = o;                                    // chunks of a file are released in order
                while (!ready[f].compare_exchange_weak(want, o + CH)) { want = o; std::this_thread::yield(); }
            } }); });
            par(F, [&](int f) { for (size_t o = 0; o < G; o += CH) {
                while (ready[f].load() < o + CH) std::this_thread::yield();
                if (pwrite(fds[f], src + (f * CH + o) % SB, CH, o) != (ssize_t)CH) perror("pwrite");
            } });
            pool.join();
            const double dt = now() - t0;
            for (int f = 0; f < F; f++) { if (maps[f]) munmap(maps[f], G); close(fds[f]); }
            printf("%-52s pass %d: %6.2f GB/s (%d allocations failed)\n",
                   mode == 0 ? "10 new files, one pwrite stream each" : mode == 1 ? "  + 5 threads MADV_POPULATE_WRITE ahead" : "  + 5 threads fallocate ahead",
                   rep, F * G / dt / 1e9, failed.load());
            fflush(stdout);
            cleanup();
        }
    rmdir(dir.c_str());
    return 0;
}
