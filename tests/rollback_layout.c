/* tests/rollback_layout.c -- sizeof/offsetof of vmig_rollback_stats as the C compiler sees include/vmig.h (compiled with
 * gcc -std=c99 -Werror and run by tests/test_rollback_host.py, which compares the line with its ctypes mirror). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("rollback_stats %zu:%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu abi=%d\n", sizeof(vmig_rollback_stats),
           offsetof(vmig_rollback_stats, files_kept), offsetof(vmig_rollback_stats, files_patched),
           offsetof(vmig_rollback_stats, files_rebuilt), offsetof(vmig_rollback_stats, files_created),
           offsetof(vmig_rollback_stats, blocks_fetched), offsetof(vmig_rollback_stats, bytes_fetched),
           offsetof(vmig_rollback_stats, files_trusted), offsetof(vmig_rollback_stats, files_read),
           offsetof(vmig_rollback_stats, bytes_read), offsetof(vmig_rollback_stats, bytes_copied),
           offsetof(vmig_rollback_stats, reserved), VMIG_ABI_VERSION);
    return 0;
}
