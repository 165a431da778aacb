/* tests/compare_layout.c -- sizeof/offsetof of vmig_compare_stats as the C compiler sees include/vmig.h (compiled with
 * gcc -std=c99 -Werror and run by tests/test_compare_host.py, which compares the line with its ctypes mirror). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("compare_stats %zu:%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu abi=%d\n", sizeof(vmig_compare_stats),
           offsetof(vmig_compare_stats, paths_added), offsetof(vmig_compare_stats, paths_removed),
           offsetof(vmig_compare_stats, paths_changed), offsetof(vmig_compare_stats, files_changed),
           offsetof(vmig_compare_stats, blocks_changed), offsetof(vmig_compare_stats, bytes_restore),
           offsetof(vmig_compare_stats, files_read), offsetof(vmig_compare_stats, bytes_read),
           offsetof(vmig_compare_stats, files_trusted), offsetof(vmig_compare_stats, files_shared),
           offsetof(vmig_compare_stats, reserved), VMIG_ABI_VERSION);
    return 0;
}
