/* tests/migrate_layer_layout.c -- sizeof/offsetof of vmig_layer_migrate_stats as the C compiler sees include/vmig.h
 * (compiled with gcc -std=c99 -Werror and run by tests/test_migrate_layer_host.py, which compares the line with its
 * ctypes mirror). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("layer_migrate_stats %zu:%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu abi=%d\n", sizeof(vmig_layer_migrate_stats),
           offsetof(vmig_layer_migrate_stats, files_trusted), offsetof(vmig_layer_migrate_stats, bytes_trusted),
           offsetof(vmig_layer_migrate_stats, files_read), offsetof(vmig_layer_migrate_stats, bytes_read),
           offsetof(vmig_layer_migrate_stats, files_unread), offsetof(vmig_layer_migrate_stats, files_verified),
           offsetof(vmig_layer_migrate_stats, bytes_verified), offsetof(vmig_layer_migrate_stats, src_recorded),
           offsetof(vmig_layer_migrate_stats, src_unrecorded), offsetof(vmig_layer_migrate_stats, reserved), VMIG_ABI_VERSION);
    return 0;
}
