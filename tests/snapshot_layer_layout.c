/* tests/snapshot_layer_layout.c -- sizeof/offsetof of vmig_layer_snapshot_stats as the C compiler sees include/vmig.h
 * (compiled with gcc -std=c99 -Werror and run by tests/test_snapshot_layer_host.py, which compares the line with its
 * ctypes mirror). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("layer_snapshot_stats %zu:%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu abi=%d\n", sizeof(vmig_layer_snapshot_stats),
           offsetof(vmig_layer_snapshot_stats, files_linked), offsetof(vmig_layer_snapshot_stats, bytes_linked),
           offsetof(vmig_layer_snapshot_stats, files_backfilled), offsetof(vmig_layer_snapshot_stats, bytes_backfilled),
           offsetof(vmig_layer_snapshot_stats, files_base_untrusted), offsetof(vmig_layer_snapshot_stats, files_trusted),
           offsetof(vmig_layer_snapshot_stats, bytes_trusted), offsetof(vmig_layer_snapshot_stats, files_read),
           offsetof(vmig_layer_snapshot_stats, bytes_read), offsetof(vmig_layer_snapshot_stats, reserved), VMIG_ABI_VERSION);
    return 0;
}
