# Builds the align_clouds oracle (orc_align_clouds.c) with the ICP and voxel oracles it calls (orc_align.c,
# orc_voxel.c); same flags as oracle/Makefile (the reference's Release defaults, -ffp-contract=off pins "no FMA").
# Test infrastructure only.
CC := /usr/bin/gcc
CFLAGS = -O3 -DNDEBUG -std=c11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

all: libouster_oracle_align_clouds.so

libouster_oracle_align_clouds.so: orc_align_clouds.c orc_align.c orc_voxel.c
	$(CC) $(CFLAGS) -shared -o $@ orc_align_clouds.c orc_align.c orc_voxel.c -lm

clean:
	rm -f libouster_oracle_align_clouds.so
