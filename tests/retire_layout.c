/* tests/retire_layout.c -- sizeof/offsetof of vmig_retire_stats as the C compiler sees include/vmig.h (compiled with
 * gcc -std=c99 -Werror and run by tests/test_retire_host.py, which compares the line with its ctypes mirror). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("retire_stats %zu:%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu abi=%d\n", sizeof(vmig_retire_stats),
           offsetof(vmig_retire_stats, versions_retired), offsetof(vmig_retire_stats, entries_removed),
           offsetof(vmig_retire_stats, files_freed), offsetof(vmig_retire_stats, bytes_freed),
           offsetof(vmig_retire_stats, records_stale), offsetof(vmig_retire_stats, records_restamped),
           offsetof(vmig_retire_stats, bytes_rehashed), offsetof(vmig_retire_stats, tables_rewritten),
           offsetof(vmig_retire_stats, reserved), VMIG_ABI_VERSION);
    return 0;
}
