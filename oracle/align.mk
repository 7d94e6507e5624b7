# Builds the cloud-to-cloud ICP oracle (orc_align.c) on its own; same flags as oracle/Makefile (the reference's
# Release defaults, -ffp-contract=off pins "no FMA").  Test infrastructure only.
CC := /usr/bin/gcc
CFLAGS = -O3 -DNDEBUG -std=c11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

all: libouster_oracle_align.so

libouster_oracle_align.so: orc_align.c
	$(CC) $(CFLAGS) -shared -o $@ orc_align.c -lm

clean:
	rm -f libouster_oracle_align.so
