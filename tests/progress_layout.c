/* tests/progress_layout.c -- sizeof/offsetof of vmig_progress and of vmig_opts.ctl as the C compiler sees include/vmig.h
 * (compared with the ctypes mirror by tests/test_cancel_host.py). */
#include <stddef.h>
#include <stdio.h>
#include "vmig.h"

int main(void)
{
    printf("progress %zu:%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu,%zu opts %zu:%zu,%zu abi=%d ecanceled=%d phases=%u,%u,%u,%u,%u,%u,%u,%u,%u\n",
           sizeof(vmig_progress), offsetof(vmig_progress, phase), offsetof(vmig_progress, running),
           offsetof(vmig_progress, bytes_total), offsetof(vmig_progress, blocks_total), offsetof(vmig_progress, bytes_hashed),
           offsetof(vmig_progress, blocks_hashed), offsetof(vmig_progress, bytes_written), offsetof(vmig_progress, bytes_verified),
           offsetof(vmig_progress, reserved), sizeof(vmig_opts), offsetof(vmig_opts, ctl), offsetof(vmig_opts, reserved),
           VMIG_ABI_VERSION, VMIG_ECANCELED, VMIG_PHASE_IDLE, VMIG_PHASE_WALK, VMIG_PHASE_DATA, VMIG_PHASE_VERIFY, VMIG_PHASE_META,
           VMIG_PHASE_PRUNE, VMIG_PHASE_TABLE, VMIG_PHASE_UNLINK, VMIG_PHASE_DONE);
    return 0;
}
