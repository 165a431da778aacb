/* tests/snapshot_layout.c -- sizeof/offsetof of vmig_snapshot_stats as the C compiler sees include/vmig.h (compiled
 * with gcc -std=c99 -Werror and run by tests/test_snapshot_host.py, which compares the line with its ctypes mirror). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("snapshot_stats %zu:%zu,%zu,%zu,%zu,%zu,%zu abi=%d\n", sizeof(vmig_snapshot_stats),
           offsetof(vmig_snapshot_stats, files_linked), offsetof(vmig_snapshot_stats, bytes_linked),
           offsetof(vmig_snapshot_stats, files_backfilled), offsetof(vmig_snapshot_stats, bytes_backfilled),
           offsetof(vmig_snapshot_stats, files_base_untrusted), offsetof(vmig_snapshot_stats, reserved), VMIG_ABI_VERSION);
    return 0;
}
