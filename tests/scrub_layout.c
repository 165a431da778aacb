/* tests/scrub_layout.c -- sizeof/offsetof of vmig_scrub_stats as the C compiler sees include/vmig.h (compiled with
 * gcc -std=c99 -Werror and run by tests/test_scrub_host.py, which compares the line with its ctypes mirror). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("scrub_stats %zu:%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu abi=%d\n", sizeof(vmig_scrub_stats),
           offsetof(vmig_scrub_stats, versions), offsetof(vmig_scrub_stats, versions_damaged),
           offsetof(vmig_scrub_stats, bytes_referenced), offsetof(vmig_scrub_stats, bytes_unique),
           offsetof(vmig_scrub_stats, files_damaged), offsetof(vmig_scrub_stats, blocks_damaged),
           offsetof(vmig_scrub_stats, files_unreadable), offsetof(vmig_scrub_stats, reserved), VMIG_ABI_VERSION);
    return 0;
}
